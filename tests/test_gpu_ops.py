"""GPU: kernel-level parity through the C ABI (the same kernels the handles launch)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import cptr, stats

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


def _rope_ref(x: torch.Tensor, pos: torch.Tensor, max_period: float = 10000.0) -> torch.Tensor:
    """rope.py:45-82 on [B, H, D] bf16 for one time step at per-row position ``pos``: interleaved pairs, fp32, -> bf16."""
    B, H, D = x.shape
    xf = x.float().view(B, H, D // 2, 2)
    freqs = torch.exp(torch.arange(D // 2, dtype=torch.float32) * (-math.log(max_period) * 2 / D))
    theta = freqs[None, :] * pos.float()[:, None]
    c, s_ = torch.cos(theta)[:, None, :], torch.sin(theta)[:, None, :]
    xr, xi = xf[..., 0], xf[..., 1]
    return torch.stack([xr * c - xi * s_, xr * s_ + xi * c], dim=-1).view(B, H, D).bfloat16()


@pytest.mark.parametrize("B,H,cap,nsplit", [(1, 32, 3000, 0), (5, 4, 3000, 1), (3, 2, 12, 0), (7, 8, 250, 3), (2, 32, 3000, 16)])
def test_fused_attention_step(lib, B, H, cap, nsplit):
    """The LM's one-launch attention step == RoPE + ring append + masked SDPA of the reference
    (transformer.py:557-597, 247-286), including a paused row and wrapped rings."""
    from moshi_b200 import _lib
    g = torch.Generator().manual_seed(B * 131 + cap)
    C = H * 128
    qkv = torch.randn(B, 3 * C, generator=g).bfloat16()
    k = torch.randn(B, H, cap, 128, generator=g).bfloat16()
    v = torch.randn(B, H, cap, 128, generator=g).bfloat16()
    pos = torch.tensor([0, 1, cap - 1, cap, 3 * cap + 5, 17, cap // 2][:B], dtype=torch.int64)
    mask = torch.ones(B, dtype=torch.bool)
    if B > 1:
        mask[1] = False                      # a paused row: no append, attends over the keys it already has
    q_in, k_in, v_in = (qkv[:, i * C:(i + 1) * C].reshape(B, H, 128) for i in range(3))
    q_rot, k_rot = _rope_ref(q_in, pos), _rope_ref(k_in, pos)
    k_ref, v_ref = k.clone(), v.clone()
    for b in range(B):
        if mask[b]:
            k_ref[b, :, pos[b] % cap] = k_rot[b]
            v_ref[b, :, pos[b] % cap] = v_in[b]
    n_valid = (pos + mask.long()).clamp(max=cap)
    allowed = torch.arange(cap)[None, :] < n_valid[:, None]
    want = F.scaled_dot_product_attention(q_rot.float()[:, :, None], k_ref.float(), v_ref.float(),
                                          allowed[:, None, None, :])[:, :, 0].reshape(B, C)
    kd, vd, out = k.cuda(), v.cuda(), torch.empty(B, C, dtype=torch.bfloat16, device="cuda")
    qd, pd, md = qkv.cuda(), pos.cuda(), mask.cuda()
    _lib.check(lib.b200_op_attn_step(cptr(qd), cptr(kd), cptr(vd), cptr(out), cptr(pd), cptr(md), B, H, cap, nsplit,
                                     10000.0, _stream()))
    torch.cuda.synchronize()
    rows = n_valid > 0                       # a paused row with an empty ring has nothing to attend to
    print(stats(f"attn step B={B} H={H} cap={cap} nsplit={nsplit}", out[rows.cuda()], want[rows]))
    torch.testing.assert_close(out.float().cpu()[rows], want[rows], rtol=2e-2, atol=2e-2)
    # ring contents: the appended key is the rotated k (one bf16 ulp of slack for sincos), untouched slots are identical
    torch.testing.assert_close(kd.cpu().float(), k_ref.float(), rtol=0, atol=4e-2)
    same = torch.ones(B, cap, dtype=torch.bool)
    for b in range(B):
        if mask[b]:
            same[b, pos[b] % cap] = False
    assert torch.equal(kd.cpu()[same[:, None].expand(B, H, cap)], k[same[:, None].expand(B, H, cap)])
    assert torch.equal(vd.cpu(), v_ref)


def _tie_free_top(B: int, card: int, n_top: int, gen: torch.Generator) -> torch.Tensor:
    """bf16 logits whose n_top largest entries are pairwise distinct (bf16 cannot hold 32000 distinct
    values in a sane range, so the bulk may tie; ties below the top-k never influence the sample)."""
    bulk = (torch.randn(B, card, generator=gen) * 1.5).clamp(-6, 3.5).bfloat16()
    # the 384 bf16 values in [4, 32): three binades x 128 mantissas
    top_vals = torch.cat([torch.arange(128, dtype=torch.float32) * s + lo for lo, s in ((4, 2 ** -5), (8, 2 ** -4), (16, 2 ** -3))])
    assert top_vals.bfloat16().float().unique().numel() == 384 and n_top <= 384
    out = bulk.clone()
    for b in range(B):
        pos = torch.randperm(card, generator=gen)[:n_top]
        vals = top_vals[torch.randperm(384, generator=gen)[:n_top]]
        out[b, pos] = vals.bfloat16()
    return out


@pytest.mark.parametrize("card,k,temp", [(2048, 250, 0.8), (32000, 25, 0.7), (64, 250, 0.8), (500, 25, 0.7),
                                         (2048, 250, 6.0), (32000, 25, 9.0)])
def test_sampler_matches_oracle(lib, card, k, temp):
    """sample_token with shared Exp(1) noise on logits whose top-(k+8) entries are tie-free."""
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
    # greedy
    _lib.check(lib.b200_op_sample(cptr(ld), None, cptr(out), B, card, 0, temp, k, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), logits.float().argmax(-1))


def test_sampler_ties_pick_lowest_index(lib):
    from moshi_b200 import _lib
    logits = torch.zeros(2, 100).bfloat16()
    logits[1, 40:] = 1.0
    out = torch.empty(2, dtype=torch.int64, device="cuda")
    ld = logits.cuda()
    _lib.check(lib.b200_op_sample(cptr(ld), None, cptr(out), 2, 100, 0, 1.0, 5, _stream()))
    torch.cuda.synchronize()
    assert out.tolist() == [0, 40]
