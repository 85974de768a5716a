"""GPU: every depformer path against the fp64 reference, at every layer and sub-step of a frame.

The depformer runs as one persistent kernel (csrc/dep_fused.cu, 3..256 sessions), as a launch chain of tensor-core GEMMs
(B200_DEPFORMER_CHAIN) or as a chain of GEMVs (one and two sessions).  After each frame the test reads
what the device computed inside the frame: ``dep_in`` (depformer_in[k] of transformer_out), every layer's per-frame cache
(``depformer.layers.<l>.k`` / ``.v``: bf16(in_proj(rmsnorm(x))) for every sub-step) and the logits, and holds each of them to
``depformer_ref64`` (tests/util.py), teacher-forced on the device's own transformer_out and tokens, under the rule whose
constants tests/test_depformer_ref_cpu.py calibrates on the bf16 oracle.  din is held to fp64 of transformer_out; the
checkpoints after it are teacher-forced on the device's own bf16 din, so that a din element the device rounded the other way
near a midpoint (correctly, within din's rule) is not counted again in every later checkpoint.  Without that, at 192 sessions
sampled (tests/test_gpu_zz_plan_runs.py), one row whose din carried 6 such flips in 1024 elements had its layer-0 k moved by
0.0044 of the rms, past layer 0's 2^-8; on the device's own din that k needs no slack at all.  A failure names the first
failing (frame, sub-step, layer, checkpoint) in the order the frame computes them.

Tokens: every sampled token must be what the reference sampler draws from the device's own logits with the same Exp(1) noise
(this checks the noise layout and the in-kernel sampler), and must equal the reference's own token unless that decision is
provably unstable under the logit difference observed on its row.

Under classifier-free guidance and with int8 linears (CASES_CHAIN) the handle always takes the launch chain, which each step's
kernel count confirms.  The checkpoints then cover all MB model rows (2B under guidance: the reference is teacher-forced on
the tokens repeated for the null half), int8 din bit for bit and the rest under the DEP_C_*_I8 constants.  The guided
``dep_logits`` and ``text_logits`` the samplers read must equal cfg_guide_bf16 of the model's own logits bit for bit (under
cfg_is_no_text the text logits are the conditioned rows), and the reference's own token comes from cfg_guide64 of its logits.

The "2b" member is the 2B model's geometry (tests/golden/moshi_dev_2b.json) with one temporal layer: the full 6-layer
depformer over dep_q 16 sub-steps, depformer_in with K 2560 and, in its sampled rows, the in-step text sampler over 48000
logits, whose indices past 32767 clear bit 15 of the sampler key's index field.

On one H100 80GB HBM3 (power limit 700 W) the whole file takes about 95 s, pytest's start-up included.  The worst ratios of
the 7B guided and int8 cases (din, k / v, logits) were 0.48, 0.59, 0.55 under guidance and 0 (exact), 0.77, 0.49 with int8;
the 2B member's fused, chain, GEMV and guided cases stayed below 0.48, 0.64 and 0.54, its int8 case (3, 33 and 129 sessions)
at 0 (exact), 0.53 and 0.58.

A value the reference rounds to bf16 near a midpoint must be rounded correctly: torch casts float64 to bf16 through float32,
which turns a value within half a float32 ulp of a midpoint into a tie.  At 129 sessions of the 2B int8 chain one row's
layer-0 RMSNorm output had its largest element at -4.828125177 (fp64), past the midpoint of -4.8125 and -4.84375 by 1.8e-7:
the handle rounded it to -4.84375, correctly, while the cast gave -4.8125.  That element is the row's int8 scale, so every
element of the row re-quantised and layer-0 k / v moved by 5.5 / 4.6 times the rule; the handle's k is bit for bit the
QLinear of the correctly rounded RMSNorm output.  tests/util.py's _bf now rounds float64 correctly.
"""
import dataclasses
import json
import pathlib

import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import LMConfig
from moshi_b200.synth import synth_lm_state_dict
from oracle.lm import sample_token
from tests.util import (cfg_guide64, cfg_guide_bf16, dep_checkpoints, dep_row_ratios, dep_row_scaled, depformer_ref64,
                        exact_row_ratios, greedy_unexcused, sample_is_stable, sampler_mismatches)

pytestmark = pytest.mark.gpu

AUTO, CHAIN, FUSED = _lib.B200_DEPFORMER_AUTO, _lib.B200_DEPFORMER_CHAIN, _lib.B200_DEPFORMER_FUSED

_2B = json.loads((pathlib.Path(__file__).parent / "golden" / "moshi_dev_2b.json").read_text())
MEMBERS = {
    # one temporal layer of the 7B shape in front of the full 7B depformer (dd 1024, 16 heads, ffn 2816, 6 layers, dep_q 8)
    "7b": LMConfig(num_layers=1, context=16),
    # 16 sub-steps (DEP_MAX_Q, the 2B model's depformer): 16 keys in the last sub-step's attention
    "q16": LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=4000, n_q=32, dep_q=16, depformer_context=16,
                    depformer_num_layers=2, delays=[0, 0] + [2] * 15 + [0] + [2] * 15),
    # ragged: ffn hidden 1000 (a K tail of 40 in linear_out, a partial 128-row tile in gate/value), card 1000, dd 512
    "ragged": LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=1000, card=1000, depformer_dim=512,
                       depformer_num_heads=8, depformer_dim_feedforward=1500, depformer_num_layers=2),
    # the 2B model (tests/golden/moshi_dev_2b.json) with one temporal layer: the full 6-layer depformer over 16 sub-steps,
    # depformer_in with K 2560 and the in-step text sampler over 48000 logits (indices past 32767)
    "2b": LMConfig.from_dict({**{k: v for k, v in _2B.items() if k not in ("conditioners", "fuser")}, "num_layers": 1,
                              "context": 16}),
}
SAMPLING = {
    "7b": dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25),
    "q16": dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25),
    "2b": dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25),
    # top-k at or above the vocabulary (1024 is the sampler's largest): the text top-k moves where the audio noise starts, the
    # clamp to card sets its width
    "ragged": dict(temp=0.8, top_k=1024, temp_text=0.7, top_k_text=1000),
}
# (member, path, depformer mode, batch sizes, of which also run with sampling).  The fused kernel's batches sit on the edges
# of its 64-session GEMM units, of the padded batch and of its 256-session limit.  No batch past 256 runs: streaming_begin
# refuses more than 256 model rows (the LM's linears take at most 256), so no handle reaches the fused kernel's limit.
CASES = [
    ("7b", "fused", AUTO, (3, 17, 63, 64, 65, 128, 129, 200, 256), (3, 129, 256)),
    ("7b", "chain", CHAIN, (3, 65, 129, 256), (65, 256)),
    ("7b", "gemv", AUTO, (1, 2), (2,)),
    ("7b", "fused-forced", FUSED, (1, 2), (1,)),
    ("q16", "fused", AUTO, (3, 65, 129), (65,)),
    ("q16", "chain", CHAIN, (3, 65, 129), (65,)),
    ("ragged", "fused", AUTO, (3, 65, 129), (3, 129)),
    ("ragged", "chain", CHAIN, (3, 65, 129), (65,)),
    ("2b", "fused", AUTO, (3, 17, 64, 65, 129, 256), (3, 129, 256)),
    ("2b", "chain", CHAIN, (3, 65, 129), (65,)),
    ("2b", "gemv", AUTO, (1, 2), (2,)),
]
# Classifier-free guidance and int8 linears: the handle builds no persistent kernel for either, so every frame runs the launch
# chain over MB model rows (2B under guidance).  Batches sit on the schedule edges of MB: GEMV up to 2 rows (4 with gemv_rows),
# stream-K up to 32, above that cluster split-K (int8) or the non-swapped kernel, the gated linear in blocks of 64 rows, more
# than 128 rows as consecutive launches.  Options: cfg (coef), no_text (cfg_is_no_text), masked (cfg_is_masked_until, the
# text logits guided too), pause (one paused row), int8 (quantize=True, on dep_row_scaled weights).
CASES_CHAIN = [
    ("7b", "cfg3-notext", (1, 2, 16, 17, 64, 65, 128), (2, 65), dict(cfg=3.0, no_text=True)),
    ("7b", "cfg1.5-masked", (3, 65), (65,), dict(cfg=1.5, masked=True, pause=1)),
    ("q16", "cfg3", (3, 65), (65,), dict(cfg=3.0, no_text=True)),
    ("ragged", "cfg3", (3, 65), (3,), dict(cfg=3.0, no_text=True)),
    ("7b", "int8", (1, 2, 3, 32, 33, 64, 65, 128, 129, 256), (3, 129), dict(int8=True)),
    ("q16", "int8", (3, 65, 129), (65,), dict(int8=True)),
    ("7b", "int8-cfg3", (3, 65), (65,), dict(int8=True, cfg=3.0, no_text=True)),
    ("2b", "cfg3-notext", (3, 65), (65,), dict(cfg=3.0, no_text=True)),
    ("2b", "int8", (3, 33, 129), (129,), dict(int8=True)),
]
FRAMES = 2                  # the second frame starts from the first frame's cache: it checks the per-frame restart


_sd_cache: dict = {}


def _state_dict(member: str, int8: bool = False) -> dict:
    if (member, int8) not in _sd_cache:
        _sd_cache.clear()
        torch.cuda.empty_cache()
        sd = synth_lm_state_dict(MEMBERS[member], seed=31, device="cuda")
        _sd_cache[(member, int8)] = dep_row_scaled(sd, seed=5) if int8 else sd
    return _sd_cache[(member, int8)]


def _model(cfg: LMConfig, sd: dict, mode: int):
    """LMModel whose depformer runs in ``mode`` (b200_lm_set_depformer)."""
    from moshi_b200.models import LMModel
    lm = LMModel(cfg, sd, device="cuda")
    _lib.check(_lib.lib().b200_lm_set_depformer(lm._h, mode))
    return lm


def _kind(kind: str, layer) -> str:
    return kind if layer is None else f"{kind}{layer}"


def _first(res: dict, frame: int, where: str, r: torch.Tensor) -> None:
    if res["first"] is None and bool((r > 1).any()):
        rows = (r > 1).nonzero().flatten().tolist()
        res["first"] = (f"frame {frame} {where}: rows {rows[:8]}{' ...' if len(rows) > 8 else ''} of {r.numel()}, "
                        f"worst ratio {float(r.max()):.3g}")


@torch.no_grad()
def _run(lm, member: str, sd: dict, B: int, sampling: bool, g: torch.Generator, opt: dict | None = None) -> dict:
    from moshi_b200.models import LMGen
    opt = opt or {}
    cfg, smp = MEMBERS[member], SAMPLING[member]
    coef = opt.get("cfg", 1.0)
    guided = coef != 1.0
    until = [b % 3 for b in range(B)] if opt.get("masked") else None
    gen = LMGen(lm, use_sampling=sampling, cfg_coef=coef, cfg_is_no_text=bool(opt.get("no_text")), cfg_is_masked_until=until,
                **smp)
    int8 = bool(opt.get("int8"))
    Q, dd, H, L, card = cfg.dep_q, cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_num_layers, cfg.card
    kt, ka = min(smp["top_k_text"], cfg.text_card), min(smp["top_k"], card)
    res = dict(worst={}, first=None, sampler=0, unexcused=0, decisions=0, differ=0, launches=[])
    lib = _lib.lib()
    with gen.streaming(B):
        MB = gen._model_batch
        if "pause" in opt:
            mask = torch.ones(B, dtype=torch.bool)
            mask[opt["pause"]] = False
            gen.set_exec_mask(mask)
        for frame in range(FRAMES):
            codes = torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g).cuda()
            noise = torch.empty(B, kt + Q * ka).exponential_(1, generator=g).cuda() if sampling else None
            n0 = lib.b200_launch_count()
            gen.step(codes, noise=noise)
            res["launches"].append(lib.b200_launch_count() - n0)
            tout = gen.read_buffer("transformer_out", torch.bfloat16, (MB, cfg.dim))
            text = gen.read_buffer("text_token", torch.int64, (B,))
            toks = gen.read_buffer("audio_tokens", torch.int64, (Q, B))
            got = dict(din=gen.read_buffer("dep_in", torch.bfloat16, (MB, Q, dd)),
                       k=[gen.read_buffer(f"depformer.layers.{l}.k", torch.bfloat16, (MB, H, Q, 64)) for l in range(L)],
                       v=[gen.read_buffer(f"depformer.layers.{l}.v", torch.bfloat16, (MB, H, Q, 64)) for l in range(L)],
                       logits=gen.read_buffer("model_dep_logits", torch.bfloat16, (Q, MB, card)))
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card))
            # the null rows are fed the conditioned rows' tokens (lm.py:826-832)
            rep = 2 if guided else 1
            want = depformer_ref64(sd, cfg, tout, text.repeat(rep), toks.repeat(1, rep), quantize=int8, din=got["din"])
            for kind, k, layer, gk, wk in dep_checkpoints(got, want):
                # int8: din is one QLinear of the bf16 transformer_out, exact given it
                r = exact_row_ratios(gk, wk) if int8 and kind == "din" else dep_row_ratios(gk, wk, kind, layer, int8)
                key = _kind(kind, layer)
                res["worst"][key] = max(res["worst"].get(key, 0.0), float(r.max()))
                _first(res, frame, f"sub-step {k} layer {layer} checkpoint {kind}", r)
            dl = got["logits"]
            if guided:
                # what the samplers read: the reference's three bf16 operations on the model's own logits, bit for bit
                mtl = gen.read_buffer("model_text_logits", torch.bfloat16, (MB, cfg.text_card))
                want_tl = mtl[:B] if opt.get("no_text") else cfg_guide_bf16(mtl, B, coef)
                _first(res, frame, "guided text logits", exact_row_ratios(tl, want_tl))
                dl = gen.read_buffer("dep_logits", torch.bfloat16, (Q, B, card))
                for k in range(Q):
                    want_dl = cfg_guide_bf16(got["logits"][k], B, coef)
                    _first(res, frame, f"sub-step {k} guided logits", exact_row_ratios(dl[k], want_dl))
            # the samplers against the reference sampler on the device's own (guided) logits and noise
            res["sampler"] += sampler_mismatches(tl, text, sampling, smp["temp_text"], smp["top_k_text"],
                                                 None if noise is None else noise[:, :kt])
            for k in range(Q):
                nk = None if noise is None else noise[:, kt + k * ka:kt + (k + 1) * ka]
                lg = dl[k]
                res["sampler"] += sampler_mismatches(lg, toks[k], sampling, smp["temp"], smp["top_k"], nk)
                # and against the reference's own (guided) token, margin-aware
                ref_lg = (cfg_guide64(want["logits"][k], B, coef) if guided else want["logits"][k].bfloat16()).float()
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


@pytest.mark.parametrize("member,path,mode,batches,sampled", CASES, ids=[f"{c[0]}-{c[1]}" for c in CASES])
def test_depformer_matches_fp64_reference(member, path, mode, batches, sampled):
    cfg = MEMBERS[member]
    sd = _state_dict(member)
    lm = _model(cfg, sd, mode)
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


@pytest.mark.parametrize("member,path,batches,sampled,opt", CASES_CHAIN, ids=[f"{c[0]}-chain-{c[1]}" for c in CASES_CHAIN])
def test_guided_and_int8_depformer_matches_fp64_reference(member, path, batches, sampled, opt):
    """The launch chain under classifier-free guidance and with int8 linears, over all MB model rows, then the guided logits the
    samplers read, bit for bit, and every token."""
    cfg = MEMBERS[member]
    int8 = bool(opt.get("int8"))
    if int8:
        cfg = dataclasses.replace(cfg, quantize=True)
    sd = _state_dict(member, int8)
    lm = _model(cfg, sd, AUTO)
    g = torch.Generator().manual_seed(len(path) * 103 + len(member))
    min_launches = cfg.dep_q * cfg.depformer_num_layers * 5      # one launch per depformer linear or attention at least
    failures = []
    try:
        for B in batches:
            for sampling in (False, True) if B in sampled else (False,):
                res = _run(lm, member, sd, B, sampling, g, opt)
                w = res["worst"]
                kv = " ".join(f"{w[f'k{l}']:.3f}/{w[f'v{l}']:.3f}" for l in range(cfg.depformer_num_layers))
                mode = "sampled" if sampling else "greedy"
                print(f"\n{member} chain-{path} B={B} {mode}: worst ratio din {w['din']:.3f}, k/v per layer {kv}, "
                      f"logits {w['logits']:.3f}; tokens differing from the reference {res['differ']}/{res['decisions']} "
                      f"({res['unexcused']} unexcused), sampler mismatches {res['sampler']}, launches per step {res['launches']}")
                if min(res["launches"]) < min_launches:
                    failures.append(f"{member} {path} B={B} {mode}: {res['launches']} launches per step, the launch chain "
                                    f"takes at least {min_launches}")
                if res["first"] is not None:
                    failures.append(f"{member} {path} B={B} {mode}: first failing {res['first']}")
                if res["unexcused"] or res["sampler"]:
                    failures.append(f"{member} {path} B={B} {mode}: {res['unexcused']} unexcused token differences, "
                                    f"{res['sampler']} sampler mismatches")
    finally:
        del lm
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)
