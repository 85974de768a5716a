"""GPU: the int8 x int8 linear (wgmma s8 x s8 -> s32) against the CPU restatement of the reference's QLinear
(oracle/quant.py; parity unpinned: bitsandbytes is absent, see that file).  Integer accumulation is exact, so the
comparison is bit for bit: quantised weights, weight scales, quantised activations, activation scales, outputs."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import quant
from tests.util import cptr, stats

pytestmark = pytest.mark.gpu

STORE, RESADD, GATE = 0, 1, 2


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gpu_linear(lib, x, w, epi, gate_rows, res=None):
    from moshi_b200 import _lib
    M, K = x.shape
    N = w.shape[0]
    tiles = torch.empty(lib.b200_op_packed_bytes_i8(N, K, epi, gate_rows), dtype=torch.uint8, device="cuda")
    sw = torch.empty(N, dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_op_quant_pack_tiles(cptr(w), cptr(tiles), cptr(sw), N, K, epi, gate_rows, _st()))
    xq = torch.empty(M, K, dtype=torch.int8, device="cuda")
    sa = torch.empty(M, dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_op_quantize_rows(cptr(x), cptr(xq), cptr(sa), M, K, _st()))
    cols = gate_rows if epi == GATE else N
    y = torch.full((M, cols), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.b200_op_linear_i8(cptr(xq), cptr(sa), cptr(tiles), cptr(sw), cptr(y), cptr(res), M, N, K, epi, gate_rows, _st()))
    torch.cuda.synchronize()
    return y, xq, sa, sw


@pytest.mark.parametrize("M,N,K", [(1, 256, 128), (3, 1024, 4096), (16, 4096, 4096), (96, 4096, 11264), (130, 2048, 1024),
                                   (256, 1024, 2816), (7, 200, 144)])
def test_int8_linear_store_is_exact(M, N, K):
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    x[0, :3] = 0.0
    y, xq, sa, sw = _gpu_linear(lib, x.cuda(), w.cuda(), STORE, 0)
    qw_o, sw_o = quant.quantize_weight(w)
    qx_o, sa_o = quant.quantize_rows(x)
    assert torch.equal(sw.cpu(), sw_o) and torch.equal(sa.cpu(), sa_o)
    assert torch.equal(xq.cpu(), qx_o)
    want = quant.qlinear(x, w)
    print(stats(f"int8 store {M}x{N}x{K}", y, want), "| vs bf16 linear:", stats("", y, (x.float() @ w.float().t())))
    assert torch.equal(y.cpu(), want)
    # and the quantised product is a faithful linear: a few percent of the output scale
    ref = x.float() @ w.float().t()
    assert (y.float().cpu() - ref).abs().max() < 0.05 * ref.abs().max() + 0.05


@pytest.mark.parametrize("M,N,K", [(5, 512, 256), (17, 4096, 4096), (96, 4096, 4096), (104, 4096, 11264), (130, 1024, 2816)])
def test_int8_linear_residual_add(M, N, K):
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M * N)
    x = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    res = torch.randn(M, N, generator=g).bfloat16()
    y, *_ = _gpu_linear(lib, x.cuda(), w.cuda(), RESADD, 0, res.cuda())
    want = (res.float() + quant.qlinear(x, w).float()).bfloat16()
    assert torch.equal(y.cpu(), want)


@pytest.mark.parametrize("M,H,K", [(2, 128, 256), (40, 2816, 1024), (96, 11264, 4096)])
def test_int8_gated_silu(M, H, K):
    """ActivationGating (gating.py:13-22) on the quantised projection: gate and value rows have their own scales."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    g = torch.Generator().manual_seed(M + H)
    x = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(2 * H, K, generator=g) / K ** 0.5).bfloat16()
    y, *_ = _gpu_linear(lib, x.cuda(), w.cuda(), GATE, H)
    h = quant.qlinear(x, w)
    want = (F.silu(h[:, :H].float()).bfloat16() * h[:, H:]).float()
    print(stats(f"int8 gate {M}x{H}x{K}", y, want))
    # silu goes through expf on the device: one bf16 ulp of slack on a handful of entries
    torch.testing.assert_close(y.float().cpu(), want, rtol=8e-3, atol=1e-3)
    assert (y.float().cpu() != want).float().mean() < 0.02


@pytest.mark.parametrize("sampling,use_graph", [(False, False), (True, True)])
def test_quantized_lm_steps_match_quantized_oracle(sampling, use_graph):
    """LMModel(quantize=True) (lm.py:107,242-243): every linear of the Temporal and Depth transformers, the depformer
    input projections and the logit heads run int8 x int8 on the tensor cores.  Each linear is exact given its input,
    so against the oracle's QLinear restatement the step differs only by the bf16 rounding noise of the other ops,
    amplified by the activation quantiser (one int8 step = absmax/127 of a row)."""
    import dataclasses

    from moshi_b200.config import tiny_lm_config
    from moshi_b200.models import LMModel
    from moshi_b200.synth import synth_lm_state_dict
    from oracle import scenarios
    from tests.test_gpu_lm import _run
    cfg = dataclasses.replace(tiny_lm_config(), quantize=True)
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    lm = LMModel(cfg, sd, device="cuda")
    m, t, _, _, worst, sm, st = _run(lm, (cfg, sd), sampling, use_graph, None, quantize=True)
    assert worst < 0.4, worst          # measured 0.25 over 41 greedy steps (bf16 model: 0.08); token agreement gated below
    if sampling:
        assert st > 0 and sm >= st - 1          # the sampler itself is exact on the GPU's own logits
    else:
        assert m / t > 0.9
    # quantisation error against the bf16 model stays small on this model (sanity: the int8 path is not garbage)
    plain = LMModel(tiny_lm_config(), sd, device="cuda")
    from moshi_b200.models import LMGen
    outs = []
    for model in (lm, plain):
        gen = LMGen(model, use_sampling=False)
        codes = scenarios.lm_input_codes(cfg, scenarios.LM_B, 1)
        with gen.streaming(scenarios.LM_B):
            gen.step(codes[0].cuda())       # first step only: later steps feed back each model's own tokens
            outs.append(gen.read_buffer("text_logits", torch.bfloat16, (scenarios.LM_B, cfg.text_card)).float().cpu())
    rel = (outs[0] - outs[1]).abs().max().item() / outs[1].abs().max().item()
    print(f"int8 vs bf16 text logits, first step: rel-to-max {rel:.3e}")
    assert rel < 0.08
