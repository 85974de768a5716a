"""GPU: the stream-K wgmma GEMM over pre-tiled weights (csrc/gemm_sk.cu) against fp32 math.

Covers the three epilogues of the LM (store, residual add, gated SiLU), ragged shapes, and work
partitions that cut tiles into many / few / no partial segments; the partition must not change the
result (partials are reduced in CTA order).  Runs late in the suite: a faulting tensor-core kernel
poisons the CUDA context for everything after it.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests.util import cptr, stats

pytestmark = pytest.mark.gpu

STORE, RESADD, GATE = 0, 1, 2


def _pack(lib, w, N, K, epi, gate_rows):
    from moshi_b200 import _lib
    nbytes = lib.b200_op_packed_bytes(N, K, epi, gate_rows)
    out = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200_op_pack_tiles(cptr(w), cptr(out), N, K, epi, gate_rows, st))
    return out


def _run(lib, x, wt, res, M, N, K, epi, gate_rows, grid=0, smem=0):
    from moshi_b200 import _lib
    cols = gate_rows if epi == GATE else N
    y = torch.full((M, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200_op_linear_sk(cptr(x), cptr(wt), cptr(y), cptr(res), M, N, K, epi, gate_rows, grid, smem, 0, st))
    torch.cuda.synchronize()
    return y


SHAPES = [(1, 512, 256), (3, 1024, 4096), (8, 12288, 4096), (16, 128, 64), (17, 4096, 11264), (96, 4096, 4096),
          (128, 2048, 1024), (200, 1024, 2816), (256, 32000, 4096), (96, 704, 256), (5, 200, 72)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_sk_store(M, N, K):
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M * 7 + N)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    wt = _pack(lib, w, N, K, STORE, 0)
    want = x.float() @ w.float().t()
    ys = {}
    for grid in (0, 37, 3, 296):
        y = _run(lib, x, wt, None, M, N, K, STORE, 0, grid=grid, smem=(100 << 10) if grid == 296 else 0)
        print(stats(f"sk store {M}x{N}x{K} grid={grid}", y, want))
        assert not torch.isnan(y.float()).any()
        torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=2e-2)
        ulp_off = ((y.float() - want.bfloat16().float()).abs() > 0).float().mean().item()
        assert ulp_off < 0.05, ulp_off
        ys[grid] = y
    # launch-to-launch reproducibility (fixed reduction order)
    again = _run(lib, x, wt, None, M, N, K, STORE, 0, grid=0)
    assert torch.equal(again, ys[0])


@pytest.mark.parametrize("M,N,K", [(1, 256, 512), (24, 4096, 4096), (96, 4096, 11264), (130, 1024, 2816), (7, 200, 72)])
def test_sk_residual_add(M, N, K):
    """x_orig + update in bf16 (transformer.py:769,777): y = res + bf16(x . w^T), in place."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    res = torch.randn(M, N, generator=g).bfloat16().cuda()
    wt = _pack(lib, w, N, K, RESADD, 0)
    want = (res.float() + (x.float() @ w.float().t()).bfloat16().float())
    for grid in (0, 11):
        y = _run(lib, x, wt, res, M, N, K, RESADD, 0, grid=grid)
        print(stats(f"sk resadd {M}x{N}x{K} grid={grid}", y, want))
        torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=3e-2)
    # in place (the LM passes y == res)
    inplace = res.clone()
    from moshi_b200 import _lib as L
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.b200_op_linear_sk(cptr(x), cptr(wt), cptr(inplace), cptr(inplace), M, N, K, RESADD, 0, 0, 0, 0, st))
    torch.cuda.synchronize()
    assert torch.equal(inplace, _run(lib, x, wt, res, M, N, K, RESADD, 0))


@pytest.mark.parametrize("M,H,K", [(1, 128, 256), (16, 11264, 4096), (96, 2816, 1024), (129, 704, 256), (200, 300, 136)])
def test_sk_gated_silu(M, H, K):
    """ActivationGating (gating.py:13-22): rows [gate ; value]; y = bf16(silu(bf16 gate)) * bf16 value."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + H)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(2 * H, K, generator=g) / K ** 0.5).bfloat16().cuda()
    wt = _pack(lib, w, 2 * H, K, GATE, H)
    h = (x.float() @ w.float().t()).bfloat16()
    want = (F.silu(h[:, :H].float()).bfloat16() * h[:, H:]).float()
    for grid in (0, 5):
        y = _run(lib, x, wt, None, M, 2 * H, K, GATE, H, grid=grid)
        print(stats(f"sk gate {M}x{H}x{K} grid={grid}", y, want))
        assert not torch.isnan(y.float()).any()
        torch.testing.assert_close(y.float(), want, rtol=2e-2, atol=3e-2)


@pytest.mark.parametrize("M,N,K,epi", [(33, 4096, 4096, RESADD), (96, 4096, 11264, RESADD), (130, 1024, 1024, STORE),
                                        (256, 2048, 1024, STORE), (96, 3072, 1024, STORE), (40, 200, 520, RESADD)])
def test_cluster_split_k(M, N, K, epi):
    """Cluster split-K (one 128-row tile per cluster, k-range per rank, DSMEM reduce-scatter): every cluster size gives
    the same bits as the whole-tile schedule up to fp32 summation order, and repeated launches are bit-identical."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M * 3 + N)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    res = torch.randn(M, N, generator=g).bfloat16().cuda() if epi == RESADD else None
    wt = _pack(lib, w, N, K, epi, 0)
    acc = (x.float() @ w.float().t())
    want = (res.float() + acc.bfloat16().float()) if epi == RESADD else acc
    for cs in (2, 4, 8):
        if (K + 63) // 64 < cs:
            continue
        y = _run(lib, x, wt, res, M, N, K, epi, 0, grid=-cs)
        print(stats(f"ck {M}x{N}x{K} epi={epi} cluster={cs}", y, want))
        assert not torch.isnan(y.float()).any()
        torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=3e-2)
        assert torch.equal(y, _run(lib, x, wt, res, M, N, K, epi, 0, grid=-cs))
    auto = _run(lib, x, wt, res, M, N, K, epi, 0, grid=0)          # what the LM launches for this shape
    torch.testing.assert_close(auto.float(), want, rtol=1e-2, atol=3e-2)


@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("N,K,epi", [(4096, 4096, STORE), (12288, 4096, STORE), (4096, 11264, RESADD), (1024, 2816, RESADD),
                                     (22528, 4096, GATE), (5632, 1024, GATE), (200, 192, STORE)])
def test_gemv_path_equals_tensor_core_path(M, N, K, epi):
    """One to four sessions: the same pre-tiled weights streamed with plain loads on the CUDA cores (gemv_kernel) against fp32
    math and against the tensor-core GEMM (both accumulate in fp32; only the summation order differs)."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M * 5 + N)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    rows = N
    w = (torch.randn(rows, K, generator=g) / K ** 0.5).bfloat16().cuda()
    gate_rows = N // 2 if epi == GATE else 0
    res = torch.randn(M, N, generator=g).bfloat16().cuda() if epi == RESADD else None
    wt = _pack(lib, w, N, K, epi, gate_rows)
    acc = x.float() @ w.float().t()
    if epi == STORE:
        want = acc
    elif epi == RESADD:
        want = res.float() + acc.bfloat16().float()
    else:
        h = acc.bfloat16()
        want = (F.silu(h[:, :gate_rows].float()).bfloat16() * h[:, gate_rows:]).float()
    before = lib.b200_op_set_gemv_max_rows(4)
    try:
        y_gemv = _run(lib, x, wt, res, M, N, K, epi, gate_rows)
        again = _run(lib, x, wt, res, M, N, K, epi, gate_rows)
        lib.b200_op_set_gemv_max_rows(0)
        y_mma = _run(lib, x, wt, res, M, N, K, epi, gate_rows)
    finally:
        lib.b200_op_set_gemv_max_rows(before)
    print(stats(f"gemv {M}x{N}x{K} epi={epi}", y_gemv, want), "| vs tensor-core path:", stats("", y_gemv, y_mma.float()))
    assert not torch.isnan(y_gemv.float()).any()
    torch.testing.assert_close(y_gemv.float(), want, rtol=2e-2, atol=3e-2)
    assert torch.equal(y_gemv, again)                                   # split partials are summed in split order
    assert ((y_gemv.float() - y_mma.float()).abs() > 0).float().mean() < 0.05      # a bf16 ulp apart now and then


def _run_ns(lib, x, wt, res, M, N, K, epi, gate_rows, cluster=0):
    from moshi_b200 import _lib
    cols = gate_rows if epi == GATE else N
    y = torch.full((M, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200_op_linear_ns(cptr(x), cptr(wt), cptr(y), cptr(res), M, N, K, epi, gate_rows, cluster, st))
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("M,N,K,epi", [(33, 4096, 4096, RESADD), (104, 12288, 4096, STORE), (96, 4096, 11264, RESADD),
                                        (128, 2048, 1024, STORE), (48, 32000, 4096, STORE), (104, 22528, 4096, GATE),
                                        (64, 5632, 1024, GATE), (40, 200, 520, RESADD), (5, 384, 72, STORE), (77, 608, 136, GATE),
                                        (104, 8192, 4096, STORE), (1, 256, 512, STORE),
                                        # above 128 sessions: two launches of up to 128 rows
                                        (130, 1024, 1024, STORE), (200, 4096, 4096, RESADD), (256, 2048, 1024, STORE), (197, 5632, 1024, GATE),
                                        (197, 12288, 4096, STORE)])
def test_ns_gemm(M, N, K, epi):
    """The non-swapped kernel (csrc/gemm_ns.cu; the LM's linears at 33..128 sessions: activations = wgmma A, two weight tiles = B,
    N = 256; two 128-session blocks above 128) against fp32 math for the three epilogues, odd tile counts, ragged N / K, every cluster size (K cut over 1..8 CTAs,
    DSMEM reduce-scatter by output columns), bit-identical repeats, and against the swap-AB kernels (same weights, same cast
    points: a bf16 ulp apart now and then from the fp32 summation order)."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M * 3 + N + epi)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    gate_rows = N // 2 if epi == GATE else 0
    cols = gate_rows if epi == GATE else N
    res = torch.randn(M, cols, generator=g).bfloat16().cuda() if epi == RESADD else None
    wt = _pack(lib, w, N, K, epi, gate_rows)
    acc = x.float() @ w.float().t()
    if epi == STORE:
        want = acc
    elif epi == RESADD:
        want = res.float() + acc.bfloat16().float()
    else:
        h = acc.bfloat16()
        want = (F.silu(h[:, :gate_rows].float()).bfloat16() * h[:, gate_rows:]).float()
    n_kb = (K + 63) // 64
    # 100 + n: single-tile units (N = 128 per instruction) with n K-splits
    for cs in ((0, 1) if epi == GATE else (0, 1, 2, 3, 4, 8, 101, 102, 104)):
        if cs % 100 > n_kb:
            continue
        y = _run_ns(lib, x, wt, res, M, N, K, epi, gate_rows, cluster=cs)
        print(stats(f"ns {M}x{N}x{K} epi={epi} cluster={cs}", y, want))
        assert not torch.isnan(y.float()).any()
        torch.testing.assert_close(y.float(), want, rtol=2e-2, atol=3e-2)
        assert torch.equal(y, _run_ns(lib, x, wt, res, M, N, K, epi, gate_rows, cluster=cs))
    # same result as the swap-AB kernels up to summation order
    from moshi_b200 import _lib as L
    y_sw = torch.full((M, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.b200_op_linear_sk(cptr(x), cptr(wt), cptr(y_sw), cptr(res), M, N, K, epi, gate_rows, 0, -1, 0, st))
    torch.cuda.synchronize()
    y = _run_ns(lib, x, wt, res, M, N, K, epi, gate_rows)
    assert ((y.float() - y_sw.float()).abs() > 0).float().mean() < 0.05
    if epi == RESADD:      # in place, as the LM calls it (y == res)
        inplace = res.clone()
        L.check(lib.b200_op_linear_ns(cptr(x), cptr(wt), cptr(inplace), cptr(inplace), M, N, K, epi, gate_rows, 0, st))
        torch.cuda.synchronize()
        assert torch.equal(inplace, y)
