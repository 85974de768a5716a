"""GPU: every depformer path against the fp64 reference, at every layer and sub-step of a frame.

The depformer runs as one persistent kernel (csrc/dep_fused.cu, 3..256 sessions), as a launch chain of tensor-core GEMMs
(B200_DEP_FUSED=0) or as a chain of GEMVs (one and two sessions).  After each frame the test reads
what the device computed inside the frame: ``dep_in`` (depformer_in[k] of transformer_out), every layer's per-frame cache
(``depformer.layers.<l>.k`` / ``.v``: bf16(in_proj(rmsnorm(x))) for every sub-step) and the logits, and holds each of them to
``depformer_ref64`` (tests/util.py), teacher-forced on the device's own transformer_out and tokens, under the rule whose
constants tests/test_depformer_ref_cpu.py calibrates on the bf16 oracle.  A failure names the first failing (frame, sub-step,
layer, checkpoint) in the order the frame computes them.

Tokens: every sampled token must be what the reference sampler draws from the device's own logits with the same Exp(1) noise
(this checks the noise layout and the in-kernel sampler), and must equal the reference's own token unless that decision is
provably unstable under the logit difference observed on its row.
"""
import os

import pytest
import torch

from moshi_b200.config import LMConfig
from moshi_b200.synth import synth_lm_state_dict
from oracle.lm import sample_token
from tests.util import (dep_checkpoints, dep_row_ratios, depformer_ref64, greedy_unexcused, sample_is_stable,
                        sampler_mismatches)

pytestmark = pytest.mark.gpu

MEMBERS = {
    # one temporal layer of the 7B shape in front of the full 7B depformer (dd 1024, 16 heads, ffn 2816, 6 layers, dep_q 8)
    "7b": LMConfig(num_layers=1, context=16),
    # 16 sub-steps (DEP_MAX_Q, the 2B model's depformer): 16 keys in the last sub-step's attention
    "q16": LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=4000, n_q=32, dep_q=16, depformer_context=16,
                    depformer_num_layers=2, delays=[0, 0] + [2] * 15 + [0] + [2] * 15),
    # ragged: ffn hidden 1000 (a K tail of 40 in linear_out, a partial 128-row tile in gate/value), card 1000, dd 512
    "ragged": LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=1000, card=1000, depformer_dim=512,
                       depformer_num_heads=8, depformer_dim_feedforward=1500, depformer_num_layers=2),
}
SAMPLING = {
    "7b": dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25),
    "q16": dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25),
    # top-k at or above the vocabulary (1024 is the sampler's largest): the text top-k moves where the audio noise starts, the
    # clamp to card sets its width
    "ragged": dict(temp=0.8, top_k=1024, temp_text=0.7, top_k_text=1000),
}
# (member, path, B200_DEP_FUSED, batch sizes, of which also run with sampling).  The fused kernel's batches sit on the edges
# of its 64-session GEMM units, of the padded batch and of its 256-session limit.  No batch past 256 runs: streaming_begin
# refuses more than 256 model rows (the LM's linears take at most 256), so no handle reaches the fused kernel's limit.
CASES = [
    ("7b", "fused", None, (3, 17, 63, 64, 65, 128, 129, 200, 256), (3, 129, 256)),
    ("7b", "chain", "0", (3, 65, 129, 256), (65, 256)),
    ("7b", "gemv", None, (1, 2), (2,)),
    ("7b", "fused-forced", "2", (1, 2), (1,)),
    ("q16", "fused", None, (3, 65, 129), (65,)),
    ("q16", "chain", "0", (3, 65, 129), (65,)),
    ("ragged", "fused", None, (3, 65, 129), (3, 129)),
    ("ragged", "chain", "0", (3, 65, 129), (65,)),
]
FRAMES = 2                  # the second frame starts from the first frame's cache: it checks the per-frame restart


_sd_cache: dict = {}


def _state_dict(member: str) -> dict:
    if member not in _sd_cache:
        _sd_cache.clear()
        torch.cuda.empty_cache()
        _sd_cache[member] = synth_lm_state_dict(MEMBERS[member], seed=31, device="cuda")
    return _sd_cache[member]


def _model(cfg: LMConfig, sd: dict, fused: str | None):
    """LMModel built with B200_DEP_FUSED = ``fused`` (None: the default), which the handle reads when it is created."""
    from moshi_b200.models import LMModel
    old = os.environ.pop("B200_DEP_FUSED", None)
    try:
        if fused is not None:
            os.environ["B200_DEP_FUSED"] = fused
        return LMModel(cfg, sd, device="cuda")
    finally:
        os.environ.pop("B200_DEP_FUSED", None)
        if old is not None:
            os.environ["B200_DEP_FUSED"] = old


def _kind(kind: str, layer) -> str:
    return kind if layer is None else f"{kind}{layer}"


@torch.no_grad()
def _run(lm, member: str, sd: dict, B: int, sampling: bool, g: torch.Generator) -> dict:
    from moshi_b200.models import LMGen
    cfg, smp = MEMBERS[member], SAMPLING[member]
    gen = LMGen(lm, use_sampling=sampling, **smp)
    Q, dd, H, L, card = cfg.dep_q, cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_num_layers, cfg.card
    kt, ka = min(smp["top_k_text"], cfg.text_card), min(smp["top_k"], card)
    res = dict(worst={}, first=None, sampler=0, unexcused=0, decisions=0, differ=0)
    with gen.streaming(B):
        for frame in range(FRAMES):
            codes = torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g).cuda()
            noise = torch.empty(B, kt + Q * ka).exponential_(1, generator=g).cuda() if sampling else None
            gen.step(codes, noise=noise)
            tout = gen.read_buffer("transformer_out", torch.bfloat16, (B, cfg.dim))
            text = gen.read_buffer("text_token", torch.int64, (B,))
            toks = gen.read_buffer("audio_tokens", torch.int64, (Q, B))
            got = dict(din=gen.read_buffer("dep_in", torch.bfloat16, (B, Q, dd)),
                       k=[gen.read_buffer(f"depformer.layers.{l}.k", torch.bfloat16, (B, H, Q, 64)) for l in range(L)],
                       v=[gen.read_buffer(f"depformer.layers.{l}.v", torch.bfloat16, (B, H, Q, 64)) for l in range(L)],
                       logits=gen.read_buffer("dep_logits", torch.bfloat16, (Q, B, card)))
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card))
            want = depformer_ref64(sd, cfg, tout, text, toks)
            for kind, k, layer, gk, wk in dep_checkpoints(got, want):
                r = dep_row_ratios(gk, wk, kind, layer)
                key = _kind(kind, layer)
                res["worst"][key] = max(res["worst"].get(key, 0.0), float(r.max()))
                if res["first"] is None and bool((r > 1).any()):
                    rows = (r > 1).nonzero().flatten().tolist()
                    res["first"] = (f"frame {frame} sub-step {k} layer {layer} checkpoint {kind}: rows {rows[:8]}"
                                    f"{' ...' if len(rows) > 8 else ''} of {B}, worst ratio {float(r.max()):.3g}")
            # the samplers against the reference sampler on the device's own logits and noise
            res["sampler"] += sampler_mismatches(tl, text, sampling, smp["temp_text"], smp["top_k_text"],
                                                 None if noise is None else noise[:, :kt])
            for k in range(Q):
                nk = None if noise is None else noise[:, kt + k * ka:kt + (k + 1) * ka]
                lg = got["logits"][k]
                res["sampler"] += sampler_mismatches(lg, toks[k], sampling, smp["temp"], smp["top_k"], nk)
                # and against the reference's own token, margin-aware
                ref_lg = want["logits"][k].bfloat16().float()
                ref_tok = sample_token(ref_lg, sampling, smp["temp"], smp["top_k"], nk, tie_break="index")
                res["decisions"] += B
                for b in (ref_tok != toks[k]).nonzero().flatten().tolist():
                    res["differ"] += 1
                    tol = float((lg[b].float() - ref_lg[b]).abs().max()) + 1e-6
                    if sampling:
                        res["unexcused"] += int(sample_is_stable(ref_lg[b:b + 1], smp["temp"], smp["top_k"], nk[b:b + 1], tol)[0])
                    else:
                        res["unexcused"] += greedy_unexcused(toks[k][b:b + 1], ref_tok[b:b + 1], ref_lg[b:b + 1].cpu(), tol)[1]
    return res


@pytest.mark.parametrize("member,path,fused,batches,sampled", CASES, ids=[f"{c[0]}-{c[1]}" for c in CASES])
def test_depformer_matches_fp64_reference(member, path, fused, batches, sampled):
    cfg = MEMBERS[member]
    sd = _state_dict(member)
    lm = _model(cfg, sd, fused)
    g = torch.Generator().manual_seed(len(path) * 101 + len(member))
    failures = []
    try:
        for B in batches:
            for sampling in (False, True) if B in sampled else (False,):
                res = _run(lm, member, sd, B, sampling, g)
                w = res["worst"]
                kv = " ".join(f"{w[f'k{l}']:.3f}/{w[f'v{l}']:.3f}" for l in range(cfg.depformer_num_layers))
                mode = "sampled" if sampling else "greedy"
                print(f"\n{member} {path} B={B} {mode}: worst ratio din {w['din']:.3f}, k/v per layer {kv}, logits {w['logits']:.3f}; "
                      f"tokens differing from the reference {res['differ']}/{res['decisions']} ({res['unexcused']} unexcused), "
                      f"sampler mismatches {res['sampler']}")
                if res["first"] is not None:
                    failures.append(f"{member} {path} B={B} {mode}: first failing {res['first']}")
                if res["unexcused"] or res["sampler"]:
                    failures.append(f"{member} {path} B={B} {mode}: {res['unexcused']} unexcused token differences, "
                                    f"{res['sampler']} sampler mismatches")
    finally:
        del lm
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)
