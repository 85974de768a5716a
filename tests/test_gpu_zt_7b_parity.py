"""GPU: BASELINE.json's own LM configuration (configs/moshi_7b_202409.json: dim 4096, 32 layers, context 3000, 32000 / 2048
vocabularies) stepped beside the CPU oracle on the same synthetic weights (VERDICT r1, "what's weak" #1).

The oracle steps the 7B model on the host cores in 1-8 s per step, so each batch size runs a handful of
teacher-synchronised steps.  Batch sizes pick the three linear schedules: 1 (GEMV kernel + chained depformer), 3 (stream-K
wgmma + fused depformer), 40 (whole-tile + cluster split-K wgmma + fused depformer).  Greedy ids are compared
margin-aware: a mismatch is excused only where the oracle's own top-2 logit gap is below twice the logit tolerance."""
import pytest
import torch

from moshi_b200.config import MOSHI_7B, LMConfig
from moshi_b200.synth import tiled_lm_state_dict
from oracle.lm import LMOracle, LMSpec
from tests.util import greedy_unexcused

pytestmark = pytest.mark.gpu

# bf16 logits after 32 layers (+ 6 depformer layers) of bf16 casts: the GPU (fp32 accumulation in registers, split-K partial sums) and
# torch's CPU kernels (their own blocking) round differently at every cast, and every rounding random-walks through the residual
# stream; for scale, the SAME session stepped by the GPU alone and inside a batch of five (another summation order, nothing
# else) differs by a comparable amount (tests/test_gpu_lm.py::test_full_size_7b_properties).  The id gate below is the strict one:
# a greedy id may only differ from the oracle's where the oracle's own top-2 gap is below twice these tolerances.
TEXT_ATOL_7B = 0.25
DEP_ATOL_7B = 0.45


@pytest.fixture(scope="module")
def seven_b():
    from moshi_b200.models import LMModel
    sd = tiled_lm_state_dict(MOSHI_7B, seed=7)
    lm = LMModel(MOSHI_7B, sd, device="cuda")
    yield sd, lm
    del lm
    torch.cuda.empty_cache()


def _sync(orc, tt, at, dep_q):
    pos = (orc.offsets % orc.cache.shape[2])
    for b in range(tt.shape[0]):
        orc.cache[b, 0, pos[b]] = tt[b]
        orc.cache[b, 1:dep_q + 1, pos[b]] = at[:, b]


def _compare(cfg, sd, lm, B, steps, seed, tol_text, tol_dep, quantize=False, prefill=None):
    from moshi_b200.models import LMGen
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, cfg.card, (steps, B, 8, 1), generator=g)
    gen = LMGen(lm, use_sampling=False)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, tie_break="index", quantize=quantize)
    orc.streaming(B)
    worst_t = worst_d = 0.0
    mism = unexc = total = 0
    with gen.streaming(B):
        if prefill is not None:
            prefill(gen, orc, g)
        for i in range(steps):
            dbg = {}
            want = orc.step(codes[i], None, None, debug=dbg)
            got = gen.step(codes[i].cuda())
            assert (want is None) == (got is None), i
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu()
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            tlo = dbg["text_logits"].float()[:, 0, 0]
            worst_t = max(worst_t, (tl - tlo).abs().max().item())
            m, u = greedy_unexcused(tt, dbg["text_token"], tlo, tol_text)
            mism += m; unexc += u; total += B
            same = tt == dbg["text_token"]
            for k in range(cfg.dep_q):                      # sub-step k is comparable while the row's earlier ids agree
                if not same.any():
                    break
                dlo = dbg["dep_logits"][k].float()[:, 0, 0]
                worst_d = max(worst_d, (dl[k] - dlo)[same].abs().max().item())
                m, u = greedy_unexcused(at[k][same], dbg["audio_tokens"][:, k][same], dlo[same], tol_dep)
                mism += m; unexc += u; total += int(same.sum())
                same = same & (at[k] == dbg["audio_tokens"][:, k])
            _sync(orc, tt, at, cfg.dep_q)
    return worst_t, worst_d, mism, unexc, total


@pytest.mark.parametrize("B,steps", [(1, 4), (3, 4), (40, 3)])
def test_7b_bf16_steps_match_the_oracle(seven_b, B, steps):
    sd, lm = seven_b
    wt, wd, mism, unexc, total = _compare(MOSHI_7B, sd, lm, B, steps, seed=100 + B, tol_text=TEXT_ATOL_7B, tol_dep=DEP_ATOL_7B)
    print(f"7B bf16, B={B}: worst text-logit diff {wt:.3e}, worst depformer-logit diff {wd:.3e}; greedy ids compared {total}, "
          f"mismatches {mism}, unexcused {unexc}")
    assert wt < TEXT_ATOL_7B and wd < DEP_ATOL_7B
    assert unexc == 0
    # random-init heads give near-uniform distributions over 32000 / 2048 candidates, so near-ties (all excused above) are common;
    # measured 88-96 % raw agreement
    assert (total - mism) / total >= 0.85


def test_7b_ring_wraps_at_3000_like_the_oracle(seven_b):
    """Positions 2998 -> 3001 with a populated ring: both sides start from the same random K/V rings and token ring, written
    through set_streaming_state's per-module entries; the new keys overwrite slots 2998, 2999, 0, 1 and the oldest keys fall out
    of the context (transformer.py:236-288, 574-585)."""
    sd, lm = seven_b
    cfg = MOSHI_7B
    B, fill = 2, 2998

    def prefill(gen, orc, g):
        H, cap, D = cfg.num_heads, cfg.context, cfg.dim // cfg.num_heads
        for li, ls in enumerate(orc.main_state.layers):
            k = (0.5 * torch.randn(B, H, cap, D, generator=g)).bfloat16()
            v = (0.5 * torch.randn(B, H, cap, D, generator=g)).bfloat16()
            ls.k.copy_(k); ls.v.copy_(v)
            ls.end_offset.fill_(fill); ls.offset.fill_(fill)
            gen._write_state(f"layers.{li}.k", k)
            gen._write_state(f"layers.{li}.v", v)
        orc.main_state.offsets.fill_(fill)
        orc.offsets.fill_(fill)
        orc.offset_cpu = fill
        ring = torch.randint(0, cfg.card, orc.cache.shape, generator=g)
        orc.cache.copy_(ring)
        gen._write_state("cache", ring)
        gen._write_state("offsets", torch.full((B,), fill, dtype=torch.int64))
        gen._write_state("model.offset", torch.full((B,), fill, dtype=torch.int64))
        from moshi_b200 import _lib
        _lib.check(gen._lib.b200_lm_set_offset_cpu(gen._h, fill))

    wt, wd, mism, unexc, total = _compare(cfg, sd, lm, B, 4, seed=9, tol_text=TEXT_ATOL_7B, tol_dep=DEP_ATOL_7B, prefill=prefill)
    print(f"7B ring wrap 2998->3001: worst text-logit diff {wt:.3e}, depformer {wd:.3e}; ids {total}, mismatches {mism}, unexcused {unexc}")
    assert wt < TEXT_ATOL_7B and wd < DEP_ATOL_7B and unexc == 0


@pytest.mark.parametrize("B,steps", [(1, 3), (3, 3), (40, 3)])
def test_7b_shapes_int8_steps_match_the_quantised_oracle(B, steps):
    """BASELINE config 5 (``LMModel(quantize=True)``: every linear an int8 QLinear) at the 7B model's real matrix shapes.  The
    CPU restatement of QLinear (oracle/quant.py: exact integer products in float64) cannot step 32 layers of them in the time
    a GPU box is worth, so this member of the family keeps every dimension of the 7B configuration (4096 / 11264 / 32000 /
    depformer 1024 / 2816 / 2048, context 3000) and cuts the depth to 4 temporal + 2 depformer layers."""
    from moshi_b200.models import LMModel
    from oracle import quant
    cfg = LMConfig.from_dict({**MOSHI_7B.to_reference_kwargs(), "num_layers": 4, "depformer_num_layers": 2, "quantize": True})
    sd = tiled_lm_state_dict(cfg, seed=11)
    lm = LMModel(cfg, sd, device="cuda")
    # the activation quantiser turns a bf16 ulp of its input into an int8 step (1/127 of the row's absmax): looser than bf16
    tol = 0.4
    wt, wd, mism, unexc, total = _compare(cfg, sd, lm, B, steps, seed=200 + B, tol_text=tol, tol_dep=tol, quantize=True)
    quant.clear_cache()
    print(f"7B-shape int8 (4+2 layers), B={B}: worst text-logit diff {wt:.3e}, depformer {wd:.3e}; ids {total}, mismatches {mism}, "
          f"unexcused {unexc}")
    assert wt < tol and wd < tol and unexc == 0
    assert (total - mism) / total >= 0.85
    del lm
    torch.cuda.empty_cache()
