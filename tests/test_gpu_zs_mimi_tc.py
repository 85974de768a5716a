"""GPU: mimi_tc_kernel (TMA + wgmma tf32 with 3xTF32 split products) at the op level: accuracy against float64, and
the conv / strided conv / dilated conv / transposed-conv geometry against torch on the reference's layouts."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests.util import cptr, stats

pytestmark = pytest.mark.gpu


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("M,N,K", [(208, 1536, 512), (208, 512, 2048), (1, 32, 32), (130, 64, 96), (4000, 128, 192), (2, 1024, 8192),
                                   (257, 2048, 512)])
def test_tc_linear_has_fp32_accuracy(M, N, K):
    """3xTF32 on the tensor cores vs an exact fp32 FMA chain, both judged against float64: the error of the split product must
    stay within a small multiple of plain fp32 matmul's (it is what the RVQ indices downstream see)."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    y = torch.full((M, N), float("nan"), device="cuda")
    _lib.check(lib.b200_op_tc_linear_f32(cptr(x), cptr(w), cptr(y), M, N, K, _stream()))
    torch.cuda.synchronize()
    want = x.double() @ w.double().t()
    torch.backends.cuda.matmul.allow_tf32 = False
    f32 = (x @ w.t()).double()
    scale = want.abs().max().item()
    err_tc = (y.double() - want).abs().max().item() / scale
    err_f32 = (f32 - want).abs().max().item() / scale
    rms_tc = ((y.double() - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt()).item()
    rms_f32 = ((f32 - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt()).item()
    print(f"tc linear {M}x{N}x{K}: max err / max|y| = {err_tc:.3e} (fp32 matmul {err_f32:.3e}); relative rms {rms_tc:.3e} (fp32 {rms_f32:.3e})")
    assert not torch.isnan(y).any()
    assert err_tc < 4e-6 and rms_tc < 2e-6          # plain TF32 would be ~5e-4


CONV_CASES = [  # cin, cout, k, stride, dil, elu, T
    (64, 32, 3, 1, 1, 1, 256), (32, 64, 1, 1, 1, 1, 256), (64, 128, 8, 4, 1, 1, 512), (128, 64, 3, 1, 2, 1, 96),
    (256, 512, 12, 6, 1, 1, 96), (512, 1024, 16, 8, 1, 1, 16), (1024, 512, 3, 1, 1, 1, 2), (512, 1024, 7, 1, 1, 0, 2),
    (128, 256, 10, 5, 1, 1, 480)]


@pytest.mark.parametrize("cin,cout,k,stride,dil,elu,T", CONV_CASES)
def test_tc_streaming_conv1d_matches_batch_conv(cin, cout, k, stride, dil, elu, T):
    """conv_test.py:63-110 pattern on the SEANet's own layer shapes: chunked streaming == one causal convolution."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    torch.manual_seed(41)
    B, chunks = 3, 3
    keff = (k - 1) * dil + 1
    P = keff - stride
    x = torch.randn(B, cin, chunks * T)
    w = torch.randn(cout, cin, k) / (cin * k) ** 0.5
    bias = torch.randn(cout)
    xin = F.elu(x) if elu else x
    want = F.conv1d(F.pad(xin.double(), (P, 0)), w.double(), bias.double(), stride=stride, dilation=dil).float()
    prev = torch.zeros(B, cin, max(P, 1), device="cuda")[:, :, :P].contiguous()
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    wd, bd = w.cuda(), bias.cuda()
    outs = []
    for c in range(chunks):
        xc = x[:, :, c * T:(c + 1) * T].contiguous().cuda()
        y = torch.full((B, cout, T // stride), float("nan"), device="cuda")
        _lib.check(lib.b200_op_tc_conv1d(cptr(xc), cptr(wd), cptr(bd), cptr(prev) if P > 0 else None, cptr(mask), cptr(y), B, cin, cout, T, k,
                                         stride, dil, elu, 0, _stream()))
        outs.append(y.cpu())
    got = torch.cat(outs, -1)
    print(stats(f"tc conv {cin}->{cout} k{k} s{stride} d{dil}", got, want))
    torch.testing.assert_close(got, want, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("cin,cout,stride,T", [(1024, 512, 8, 2), (512, 256, 6, 16), (256, 128, 5, 96), (128, 64, 4, 480)])
def test_tc_streaming_convtr1d_matches_batch(cin, cout, stride, T):
    """StreamingConvTranspose1d (conv.py:340-362) as two taps over [x[t-1], x[t]]: chunked streaming == one transposed
    convolution with the trailing K - S samples cut (the causal trim of the non-streaming path)."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    torch.manual_seed(43)
    B, chunks, k = 2, 3, 2 * stride
    x = torch.randn(B, cin, chunks * T)
    w = torch.randn(cin, cout, k) / (2 * cin) ** 0.5
    bias = torch.randn(cout)
    xin = F.elu(x)
    full = F.conv_transpose1d(xin.double(), w.double(), bias.double(), stride=stride).float()
    want = full[..., :chunks * T * stride]
    prev = torch.zeros(B, cin, 1, device="cuda")
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    wd, bd = w.cuda(), bias.cuda()
    outs = []
    for c in range(chunks):
        xc = x[:, :, c * T:(c + 1) * T].contiguous().cuda()
        y = torch.full((B, cout, T * stride), float("nan"), device="cuda")
        _lib.check(lib.b200_op_tc_conv1d(cptr(xc), cptr(wd), cptr(bd), cptr(prev), cptr(mask), cptr(y), B, cin, cout, T, k, stride, 1, 1, 1,
                                         _stream()))
        outs.append(y.cpu())
    got = torch.cat(outs, -1)
    print(stats(f"tc convtr {cin}->{cout} s{stride}", got, want))
    torch.testing.assert_close(got, want, rtol=2e-5, atol=2e-5)
