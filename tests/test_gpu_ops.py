"""GPU: kernel-level parity through the C ABI (the same kernels the handles launch)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests.util import (ATTN_C, ATTN_REL, attn_err_ratio, attn_ref64, attn_scenario, cptr, dep_scenario, rmsnorm_ref64, rmsnorm_verdict,
                        stats)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    return _lib.lib()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("M,N,K", [(1, 512, 256), (3, 1024, 4096), (8, 12288, 4096), (17, 4096, 11264),
                                   (96, 4096, 4096), (128, 2048, 1024), (200, 1024, 2816), (5, 200, 72)])
def test_linear_bf16(lib, M, N, K):
    """The LM's linear on row-major weights (packed on the fly): GEMV kernel at M <= 2, wgmma kernels above."""
    from moshi_b200 import _lib
    g = torch.Generator().manual_seed(M * 7 + N)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().cuda()
    y = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.b200_op_linear_bf16(cptr(x), cptr(w), cptr(y), M, N, K, _stream()))
    torch.cuda.synchronize()
    want = (x.float() @ w.float().t())
    print(stats(f"linear {M}x{N}x{K}", y, want))
    assert not torch.isnan(y.float()).any()
    # bf16 output rounding: half an ulp of the result plus fp32 accumulation-order noise
    torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=2e-2)
    # exactness up to one bf16 ulp for almost all entries
    ulp_off = ((y.float() - want.bfloat16().float()).abs() > 0).float().mean().item()
    assert ulp_off < 0.05, ulp_off


@pytest.mark.parametrize("cin,cout,k,stride,dil,elu", [(1, 64, 7, 1, 1, 0), (64, 32, 3, 1, 1, 1), (32, 64, 1, 1, 1, 1),
                                                       (64, 128, 8, 4, 1, 1), (128, 64, 3, 1, 2, 1), (512, 1024, 16, 8, 1, 1),
                                                       (20, 24, 4, 2, 1, 0)])
def test_streaming_conv1d_matches_batch_conv(lib, cin, cout, k, stride, dil, elu):
    """conv_test.py:63-110 pattern: chunked streaming == one causal convolution over the whole signal."""
    from moshi_b200 import _lib
    torch.manual_seed(41)
    B, chunks, T = 3, 4, 8 * stride
    keff = (k - 1) * dil + 1
    P = keff - stride
    x = torch.randn(B, cin, chunks * T)
    w = torch.randn(cout, cin, k) / (cin * k) ** 0.5
    bias = torch.randn(cout)
    xin = F.elu(x) if elu else x
    want = F.conv1d(F.pad(xin, (P, 0)), w, bias, stride=stride, dilation=dil)
    prev = torch.zeros(B, cin, max(P, 1), device="cuda")
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    wd, bd = w.cuda(), bias.cuda()      # keep the device tensors alive across the call
    outs = []
    for c in range(chunks):
        xc = x[..., c * T:(c + 1) * T].contiguous().cuda()
        y = torch.empty(B, cout, T // stride, device="cuda")
        _lib.check(lib.b200_op_conv1d(cptr(xc), cptr(wd), cptr(bd), cptr(prev), cptr(mask), cptr(y),
                                      B, cin, cout, T, k, stride, dil, elu, _stream()))
        outs.append(y.cpu())
    got = torch.cat(outs, -1)
    print(stats(f"conv1d {cin}->{cout} k{k} s{stride} d{dil}", got, want))
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_streaming_conv1d_exec_mask_freezes_state(lib):
    from moshi_b200 import _lib
    torch.manual_seed(0)
    B, cin, cout, k, T = 2, 16, 16, 3, 8
    w, bias = torch.randn(cout, cin, k).cuda(), torch.randn(cout).cuda()
    prev = torch.randn(B, cin, k - 1, device="cuda")
    before = prev.clone()
    mask = torch.tensor([True, False], device="cuda")
    x = torch.randn(B, cin, T, device="cuda")
    y = torch.empty(B, cout, T, device="cuda")
    _lib.check(lib.b200_op_conv1d(cptr(x), cptr(w), cptr(bias), cptr(prev), cptr(mask), cptr(y), B, cin, cout, T, k, 1, 1, 0,
                                  _stream()))
    assert torch.equal(prev[1], before[1])
    assert torch.equal(prev[0], x[0, :, -2:])


def _attn_launch(lib, sc: dict, k, v, nsplit: int) -> torch.Tensor:
    from moshi_b200 import _lib
    out = torch.full((sc["B"], sc["H"] * 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    qd, pd, md = sc["qkv"].cuda(), sc["pos"].cuda(), sc["mask"].cuda()
    _lib.check(lib.b200_op_attn_step(cptr(qd), cptr(k), cptr(v), cptr(out), cptr(pd), cptr(md), sc["B"], sc["H"], sc["cap"], nsplit,
                                     10000.0, _stream()))
    torch.cuda.synchronize()
    return out


def _check_attn_step(lib, sc: dict, nsplit: int, label: str) -> None:
    """One step of the kernel on a scenario of tests.util.attn_scenario: outputs against attn_ref64, the ring it leaves behind
    against the reference ring."""
    kd, vd = sc["k"].cuda(), sc["v"].cuda()
    out = _attn_launch(lib, sc, kd, vd, nsplit)
    k_got, v_got = kd.cpu(), vd.cpu()
    # the reference attends over the key the kernel appended (checked below against the fp32-RoPE key on its own)
    want = attn_ref64(sc["q_rot"], k_got, sc["v_ref"], sc["n_valid"])
    ratio = attn_err_ratio(out, want)
    print(f"{label}: B={sc['B']} nsplit={sc['nsplit']}: worst |err| / tolerance {ratio:.3f} "
          f"(tolerance {ATTN_REL:.3g} |want| + {ATTN_C:.3g} rms)")
    assert torch.isfinite(out.float()).all()
    assert ratio <= 1.0
    # ring contents: untouched slots keep their bits (NaN poison included), values are appended bit for bit
    B, H, cap = sc["B"], sc["H"], sc["cap"]
    same = torch.ones(B, cap, dtype=torch.bool)
    for b in range(B):
        if sc["mask"][b]:
            same[b, int(sc["pos"][b]) % cap] = False
    keep = same[:, None].expand(B, H, cap)
    assert torch.equal(k_got.view(torch.int16)[keep], sc["k"].view(torch.int16)[keep])
    assert torch.equal(v_got.view(torch.int16), sc["v_ref"].view(torch.int16))
    # the appended key: the fp32-RoPE reference within one bf16 ulp of the head's largest element (an angle that differs in
    # the last bits of fp32 moves small elements by more than their own ulp), on >= 99 % of the elements exactly
    new = ~keep
    got_k = k_got.permute(0, 2, 1, 3)[new.permute(0, 2, 1)].float()
    want_k = sc["k_ref"].permute(0, 2, 1, 3)[new.permute(0, 2, 1)].float()
    top = want_k.abs().amax(-1, keepdim=True)
    ulp = 2.0 ** (torch.floor(torch.log2(top)) - 7)
    assert ((got_k - want_k).abs() <= ulp).all(), ((got_k - want_k).abs() / ulp).max()
    assert (got_k == want_k).float().mean() >= 0.99, (got_k == want_k).float().mean()


@pytest.mark.parametrize("nsplit", [1, 2, 3, 5, 16, 0])
@pytest.mark.parametrize("cap", [3000, 250, 12])
@pytest.mark.parametrize("H", [32, 20, 2])
def test_fused_attention_step(lib, H, cap, nsplit):
    """The LM's one-launch attention step == RoPE + ring append + attention over the valid slots (transformer.py:557-597,
    247-286) in fp64, on the rows of tests.util.attn_scenario: fills at the group / loop-step / split edges, wrapped rings
    (one hour at 12.5 Hz), paused rows, needles on every split edge and on the key the step overwrites,
    NaN poison past the fill.  nsplit 0 is the LM's own choice."""
    _check_attn_step(lib, attn_scenario(H, cap, nsplit), nsplit, f"attn step H={H} cap={cap}")


@pytest.mark.parametrize("H,cap,nsplit,qk_scale,v_scale", [(20, 250, 5, 16.0, 1.0), (2, 12, 3, 16.0, 1.0)] + [
    (H, cap, ns, qk, v) for H, cap, ns in [(32, 3000, 0), (32, 3000, 16), (20, 250, 5)] for qk, v in [(1e-3, 1.0), (1.0, 1e3)]])
def test_fused_attention_step_magnitudes(lib, H, cap, nsplit, qk_scale, v_scale):
    """q and k x16 (the softmax is nearly one-hot), x1e-3 (nearly uniform), v x1e3; no needles, so every key counts.
    x16 stays at short rings: there one bf16 ulp of a rotated query element, which the kernel's fp32 RoPE and the host's
    round differently now and then, moves a score by ~0.1, and among 3000 keys two of them are that close."""
    sc = attn_scenario(H, cap, nsplit, qk_scale=qk_scale, v_scale=v_scale, needles=False, seed=1)
    _check_attn_step(lib, sc, nsplit, f"attn step H={H} cap={cap} q,k x{qk_scale:g} v x{v_scale:g}")


@pytest.mark.parametrize("H", [16, 2])
@pytest.mark.parametrize("B", [1, 3, 80])
@pytest.mark.parametrize("dep_q", [8, 16])
def test_depformer_attention_step(lib, B, H, dep_q):
    """dep_attn_step_kernel through sub-steps 0..dep_q - 1 of one frame: the new k / v land in row `step` of the cache bit for
    bit, the query attends over rows 0..step (fp64 reference, needles on key 0 and key `step`), and the NaN poison of the
    rows after `step` is neither read nor changed."""
    from moshi_b200 import _lib
    sc = dep_scenario(B, H, dep_q)
    D, C = 64, H * 64
    kc = torch.full((B, H, dep_q, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    qkv = sc["qkv"].cuda()
    worst = 0.0
    for s in range(dep_q):
        out = torch.full((B, C), float("nan"), dtype=torch.bfloat16, device="cuda")
        _lib.check(lib.b200_op_dep_attn_step(cptr(qkv[s]), cptr(kc), cptr(vc), cptr(out), B, H, dep_q, s, _stream()))
        torch.cuda.synchronize()
        assert torch.isfinite(out.float()).all(), s
        r = attn_err_ratio(out, sc["want"][s])
        worst = max(worst, r)
        assert r <= 1.0, (s, r)
        k_got, v_got = kc.cpu(), vc.cpu()
        assert torch.equal(k_got[:, :, :s + 1].view(torch.int16), sc["k"][:, :, :s + 1].view(torch.int16)), s
        assert torch.equal(v_got[:, :, :s + 1].view(torch.int16), sc["v"][:, :, :s + 1].view(torch.int16)), s
        assert torch.isnan(k_got[:, :, s + 1:].float()).all() and torch.isnan(v_got[:, :, s + 1:].float()).all(), s
    print(f"dep attn B={B} H={H} dep_q={dep_q}: worst |err| / tolerance {worst:.3f}")
    assert lib.b200_op_dep_attn_step(cptr(qkv[0]), cptr(kc), cptr(vc), cptr(out), B, H, 17, 0, _stream()) == _lib.B200_ERR_SHAPE


def _norm_rows(M: int, dim: int, g: torch.Generator) -> torch.Tensor:
    """randn rows, rows x1e-3 and x1e4, one outlier channel at 2000 in a unit row, an all-zero row (cycled over M)."""
    x = torch.randn(M, dim, generator=g)
    for m in range(M):
        kind = m % 5
        if kind == 1:
            x[m] *= 1e-3
        elif kind == 2:
            x[m] *= 1e4
        elif kind == 3:
            x[m, (m * 37) % dim] = 2000.0
        elif kind == 4:
            x[m] = 0.0
    return x.bfloat16()


def _norm_alpha(dim: int, g: torch.Generator) -> torch.Tensor:
    alpha = torch.randn(dim, generator=g) + 0.5                         # negatives included
    alpha[::17] = 0.0
    return alpha.bfloat16()


@pytest.mark.parametrize("M", [3, 40, 130])
@pytest.mark.parametrize("dim", [4096, 2560, 1024, 256])
def test_rmsnorm_kernel(lib, M, dim):
    """rmsnorm_kernel (transformer.py:45-58, eps 1e-8): every element within one bf16 ulp of bf16(fp64 RMSNorm), >= 99.9 %
    exact; an all-zero row gives zeros, not NaN."""
    from moshi_b200 import _lib
    g = torch.Generator().manual_seed(M * 3 + dim)
    x, alpha = _norm_rows(M, dim, g), _norm_alpha(dim, g)
    xd, ad = x.cuda(), alpha.cuda()
    y = torch.full((M, dim), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.b200_op_rmsnorm(cptr(xd), cptr(ad), cptr(y), M, dim, _stream()))
    torch.cuda.synchronize()
    ulps, exact = rmsnorm_verdict(y, x, alpha)
    print(f"rmsnorm M={M} dim={dim}: worst {ulps:.0f} ulp (tolerance 1), {exact:.5f} exact (tolerance 0.999)")
    assert ulps <= 1 and exact >= 0.999
    zero = (x.float() == 0).all(-1)
    assert torch.equal(y.cpu()[zero].float(), torch.zeros_like(y.cpu()[zero].float()))


@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("dim", [4096, 2560, 1024, 256])
@pytest.mark.parametrize("epi", [0, 1, 2])
def test_gemv_with_folded_rmsnorm(lib, M, dim, epi):
    """The RMSNorm folded into the GEMV's activation staging (norm_linear at one or two sessions) against fp64
    epi(bf16(rmsnorm_ref64(x)) . W^T), with the GEMV test's tolerances; above the GEMV rows the entry point refuses."""
    from moshi_b200 import _lib
    from tests.test_gpu_zy_sk_gemm import _pack
    g = torch.Generator().manual_seed(M * 11 + dim + epi)
    N = 1024 if epi != 2 else 2048
    gate_rows = N // 2 if epi == 2 else 0
    x, alpha = _norm_rows(M, dim, g), _norm_alpha(dim, g)
    w = (torch.randn(N, dim, generator=g) / dim ** 0.5).bfloat16()
    res = torch.randn(M, N, generator=g).bfloat16() if epi == 1 else None
    xn = rmsnorm_ref64(x, alpha).bfloat16()
    acc = xn.double() @ w.double().t()
    if epi == 0:
        want = acc
    elif epi == 1:
        want = res.double() + acc.bfloat16().double()
    else:
        h = acc.bfloat16()
        want = (F.silu(h[:, :gate_rows].float()).bfloat16() * h[:, gate_rows:]).double()
    xd, ad, wd = x.cuda(), alpha.cuda(), w.cuda()
    rd = res.cuda() if res is not None else None
    wt = _pack(lib, wd, N, dim, epi, gate_rows)
    cols = gate_rows if epi == 2 else N
    y = torch.full((M, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    before = lib.b200_op_set_gemv_max_rows(4)
    try:
        _lib.check(lib.b200_op_linear_sk_norm(cptr(xd), cptr(ad), cptr(wt), cptr(y), cptr(rd), M, N, dim, epi, gate_rows, _stream()))
        torch.cuda.synchronize()
        lib.b200_op_set_gemv_max_rows(M - 1)
        rc = lib.b200_op_linear_sk_norm(cptr(xd), cptr(ad), cptr(wt), cptr(y), cptr(rd), M, N, dim, epi, gate_rows, _stream())
    finally:
        lib.b200_op_set_gemv_max_rows(before)
    assert rc == _lib.B200_ERR_STATE
    print(stats(f"gemv + rmsnorm M={M} dim={dim} epi={epi}", y, want.float()))
    assert torch.isfinite(y.float()).all()
    torch.testing.assert_close(y.float().cpu(), want.float(), rtol=2e-2, atol=3e-2)


def _tie_free_top(B: int, card: int, n_top: int, gen: torch.Generator, lo_index: int = 0) -> torch.Tensor:
    """bf16 logits whose n_top largest entries are pairwise distinct (bf16 cannot hold 32000 distinct
    values in a sane range, so the bulk may tie; ties below the top-k never influence the sample), placed at indices
    >= ``lo_index``."""
    # the 384 bf16 values in [4, 32): three binades x 128 mantissas; for more, the 1152 in [1/16, 32) above a lower bulk
    nb, bulk_hi = (3, 3.5) if n_top <= 384 else (9, 0.06)
    bulk = (torch.randn(B, card, generator=gen) * 1.5).clamp(-6, bulk_hi).bfloat16()
    top_vals = torch.cat([torch.arange(128, dtype=torch.float32) * 2.0 ** (e - 7) + 2.0 ** e for e in range(5 - nb, 5)])
    assert top_vals.bfloat16().float().unique().numel() == 128 * nb and n_top <= 128 * nb
    out = bulk.clone()
    for b in range(B):
        pos = lo_index + torch.randperm(card - lo_index, generator=gen)[:n_top]
        vals = top_vals[torch.randperm(top_vals.numel(), generator=gen)[:n_top]]
        out[b, pos] = vals.bfloat16()
    return out


def _edge_rows(card: int, k: int, gen: torch.Generator) -> torch.Tensor:
    """Three bf16 logit rows [3, card]: six equal logits across the k-th place (ranks k-3 .. k+2; at the top when k is 1);
    +inf on the sixth-ranked token and -inf on the top one; -inf on the top token alone."""
    base = _tie_free_top(1, card, min(card, k + 8), gen)[0]
    srt = torch.sort(base.float(), descending=True, stable=True).indices
    tie, inf, ninf = base.clone(), base.clone(), base.clone()
    lo, hi = max(0, k - 3), min(card, k + 3)
    tie[srt[lo:hi]] = base[srt[lo]]
    inf[srt[5]] = float("inf")
    inf[srt[0]] = float("-inf")
    ninf[srt[0]] = float("-inf")
    return torch.stack([tie, inf, ninf])


def _high_index_rows(card: int, k: int, gen: torch.Generator) -> torch.Tensor:
    """Four bf16 logit rows [4, card] for vocabularies past 32768, where the kernel's sort key holds the index as 0xFFFF - i
    and indices >= 32768 clear bit 15 of that field: the top-(k+8) entirely at indices >= 32768; a tie at the top across
    32767 / 32768 (the lower index wins); the same tie at the k-th place; the top-(k+8) at >= 32768 with a tie at the top
    between 32768 and the last index."""
    rows = _tie_free_top(4, card, min(card - 32768, k + 8), gen, lo_index=32768)
    top = float(rows.float().max()) * 2
    rows[1, [32767, 32768]] = top
    kth = torch.sort(rows[2].float(), descending=True, stable=True).values[k - 1]
    rows[2, [32767, 32768]] = kth.bfloat16()
    rows[3, [32768, card - 1]] = top
    return rows


@pytest.mark.parametrize("card,k,temp", [(2048, 250, 0.8), (32000, 25, 0.7), (64, 250, 0.8), (500, 25, 0.7),
                                         (2048, 250, 6.0), (32000, 25, 9.0), (2048, 1, 0.8), (2048, 250, 1e-3),
                                         (32000, 25, 1e-3), (48000, 25, 0.7), (48000, 1024, 0.8), (48000, 1, 0.7)])
def test_sampler_matches_oracle(lib, card, k, temp):
    """sample_token with shared Exp(1) noise on logits whose top-(k+8) entries are tie-free, then on the edge rows of
    ``_edge_rows`` (and past 32768 tokens those of ``_high_index_rows``) against the reference sampler with ties ranked by
    index (the order the kernel defines), sampled and greedy.  With k = 1 the sample is the greedy token."""
    from moshi_b200 import _lib
    from oracle.lm import sample_token
    g = torch.Generator().manual_seed(3)
    B = 33
    kk = min(k, card)
    logits = _tie_free_top(B, card, min(card, kk + 8), g)
    noise = torch.empty(B, kk).exponential_(1, generator=g)
    want = sample_token(logits.float()[:, None, None, :], True, temp, k, noise)[:, 0, 0]
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    ld, nd = logits.cuda(), noise.cuda()
    _lib.check(lib.b200_op_sample(cptr(ld), cptr(nd), cptr(out), B, card, 1, temp, k, _stream()))
    torch.cuda.synchronize()
    agree = (out.cpu() == want).float().mean().item()
    print(f"sampler card={card} k={k} temp={temp}: agreement {agree:.3f}, distinct winners {want.unique().numel()}")
    assert agree == 1.0
    if k == 1:
        assert torch.equal(out.cpu(), logits.float().argmax(-1))
    # edge rows
    edge = _edge_rows(card, kk, g)
    en = torch.empty(edge.shape[0], kk).exponential_(1, generator=g)
    ewant = sample_token(edge.float(), True, temp, k, en, tie_break="index")
    eout = torch.empty(edge.shape[0], dtype=torch.int64, device="cuda")
    ed, end = edge.cuda(), en.cuda()
    _lib.check(lib.b200_op_sample(cptr(ed), cptr(end), cptr(eout), edge.shape[0], card, 1, temp, k, _stream()))
    torch.cuda.synchronize()
    print(f"  edge rows (ties at the k-th place, +inf / -inf, -inf): got {eout.tolist()}, want {ewant.tolist()}")
    assert torch.equal(eout.cpu(), ewant)
    if k == 1:
        assert torch.equal(eout.cpu(), edge.float().argmax(-1))
    # greedy
    _lib.check(lib.b200_op_sample(cptr(ld), None, cptr(out), B, card, 0, temp, k, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), logits.float().argmax(-1))
    if card <= 32768:
        return
    high = _high_index_rows(card, kk, g)
    hn = torch.empty(high.shape[0], kk).exponential_(1, generator=g)
    hd, hnd = high.cuda(), hn.cuda()
    for sampling in (1, 0):
        hwant = sample_token(high.float(), bool(sampling), temp, k, hn, tie_break="index")
        hout = torch.empty(high.shape[0], dtype=torch.int64, device="cuda")
        _lib.check(lib.b200_op_sample(cptr(hd), cptr(hnd) if sampling else None, cptr(hout), high.shape[0], card, sampling,
                                      temp, k, _stream()))
        torch.cuda.synchronize()
        print(f"  rows past index 32767 ({'sampled' if sampling else 'greedy'}): got {hout.tolist()}, want {hwant.tolist()}")
        assert torch.equal(hout.cpu(), hwant)
    assert high.float()[[1, 3]].argmax(-1).tolist() == [32767, 32768]          # the rows hold the ties they are built for


def test_sampler_ties_pick_lowest_index(lib):
    from moshi_b200 import _lib
    logits = torch.zeros(2, 100).bfloat16()
    logits[1, 40:] = 1.0
    out = torch.empty(2, dtype=torch.int64, device="cuda")
    ld = logits.cuda()
    _lib.check(lib.b200_op_sample(cptr(ld), None, cptr(out), 2, 100, 0, 1.0, 5, _stream()))
    torch.cuda.synchronize()
    assert out.tolist() == [0, 40]
