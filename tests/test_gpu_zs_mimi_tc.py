"""GPU: mimi_tc_kernel (TMA + wgmma tf32 with 3xTF32 split products) at the op level, on the inputs no plan run of
tests/test_gpu_zz_mimi_plan_runs.py covers: flat token rows (b200_op_tc_linear_f32, whose last 128-row tile is partial), the
transposed convs at 2 sessions over two chunks, and a dilated conv (the default configuration has none).  Every output is
held to the per-output fp64 rule of tests/util.py (tc_ratios) at its tightest constant, TC_C."""
import ctypes as C

import pytest
import torch

from tests.test_gpu_zz_mimi_plan_runs import tc_conv_case
from tests.util import TC_C, TC_CONV, TC_CONVTR, TC_LINEAR, cptr, tc_ratios, tc_ref64

pytestmark = pytest.mark.gpu


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("M,N,K", [(208, 1536, 512), (208, 512, 2048), (1, 32, 32), (130, 64, 96), (4000, 128, 192), (2, 1024, 8192),
                                   (257, 2048, 512)])
def test_tc_linear_has_fp32_accuracy(M, N, K):
    """y = x . w^T on flat rows (one session of M rows on 128 x 1 tiles): every output within the fp64 rule, none left NaN."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    y = torch.full((M, N), float("nan"), device="cuda")
    _lib.check(lib.b200_op_tc_linear_f32(cptr(x), cptr(w), cptr(y), M, N, K, _stream()))
    torch.cuda.synchronize()
    want, scale = tc_ref64(TC_LINEAR, x, w)
    r = tc_ratios(y, want, scale)
    print(f"tc linear {M}x{N}x{K}: worst ratio {float(r.max()):.3g}, TC_C needed {float(r.max()) * TC_C:.3g}")
    assert not torch.isnan(y).any()
    assert float(r.max()) <= 1


@pytest.mark.parametrize("cin,cout,stride,T", [(1024, 512, 8, 2), (512, 256, 6, 16), (256, 128, 5, 96), (128, 64, 4, 480)])
def test_tc_streaming_convtr1d_matches_batch(cin, cout, stride, T):
    """StreamingConvTranspose1d (conv.py:340-362) as two taps over [x[t-1], x[t]], 2 sessions, two chunks carrying x[-1], the
    second with session 1 paused."""
    from moshi_b200 import _lib
    layer = dict(kind=TC_CONVTR, cin=cin, cout=cout, k=2 * stride, stride=stride, dil=1, elu=True)
    g = torch.Generator(device="cuda").manual_seed(43 + cin)
    need, bad = tc_conv_case(_lib.lib(), layer, 2, T, g, 1, f"tc convtr {cin}->{cout} s{stride}", TC_C)
    print(f"tc convtr {cin}->{cout} s{stride}: TC_C needed {need:.3g}")
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("B", [3, 65])
def test_tc_dilated_conv1d(B):
    """A residual conv of encoder.4's shape at dilation 2 (128 -> 64, 3 taps, 4 carried steps), two chunks."""
    from moshi_b200 import _lib
    layer = dict(kind=TC_CONV, cin=128, cout=64, k=3, stride=1, dil=2, elu=True)
    g = torch.Generator(device="cuda").manual_seed(41 + B)
    need, bad = tc_conv_case(_lib.lib(), layer, B, 96 * 5, g, B - 1, f"tc conv dilation 2 B={B}", TC_C)
    print(f"tc conv dilation 2 B={B}: TC_C needed {need:.3g}")
    assert not bad, "\n".join(bad)
