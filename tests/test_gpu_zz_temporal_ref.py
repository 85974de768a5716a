"""GPU: every layer of the temporal transformer against the fp64 reference, teacher-forced on per-layer taps, at serving batch
and for every linear schedule; then the same steps without taps, bit for bit.

With ``b200_lm_set_taps`` on, each step also copies the summed embeddings and, per layer, the attention output, x after the
attention residual, the gated hidden and x after the MLP residual.  The test holds the embeddings (bit for bit), then every layer's new k
and v (read from the rings at the step's slot), attn_out, x_attn, gated and x_out, then transformer_out, the model's text
logits and dep_in, to ``temporal_*_ref64`` (tests/util.py) under the rule whose constants tests/test_temporal_ref_cpu.py
calibrates on the bf16 oracle.  Each reference layer starts from the device's own input of that layer, so each linear is
judged on its own input and the bound does not grow with depth.  Under quantize=True x_attn and x_out must be bit-exact.  A
failure names the first failing (step, layer, checkpoint, rows).  Paused rows must leave their ring slot and position alone.

The same inputs then run again from a fresh streaming_begin with the taps off and the step graph on: ring entries,
transformer_out, text logits, dep_in and every token must be bit-identical.  The taps change which kernels are adjacent for
programmatic dependent launch, so this extends the per-layer verdict to the launch chain the benchmark runs.

The rings hold random history (positions written per row, a few hundred frames in), sized by kv_capacity so that 256
sessions fit.  Batches pick the linear schedules: 1-2 rows GEMV (RMSNorm folded in), 3-32 swap-AB stream-K, 33-128 the
non-swapped kernel, 129-256 that kernel as two 128-row blocks; int8 takes cluster split-K above 32 rows.

Besides the 7B model and its 4-layer member, the cases cover the 2B model (tests/golden/moshi_dev_2b.json: dim 2560, 20
heads, ffn 7040, RoPE period 1e5, 33 embedding tables, text head N 48000, depformer_in 16 x 1024), all 24 layers and a 4-layer
member in bf16 and int8, under guidance with a condition sum, paged, and an hour into a session (position 45 000, the ring
wrapped); and an STT geometry (dim 2048, 16 heads, dep_q 0, 32 user streams, four extra heads of six, stepped with
step_with_extra_heads), whose extra heads are held to extra_heads_ref64 on every row.  The embeddings are held bit for bit to
temporal_embed_bf16, the reference's chain of bf16 adds (the fp64 rule's headroom there depends on the tables' values).

On one H100 80GB HBM3 (power limit 700 W) the whole file takes about 100 s, building the models included (the 2B and STT
cases about 25 s of it).  The worst ratios it met (1 = at the tolerance) were 0.74 at k, 0.55 at v, 0.55 at attn_out, 0.53
at x_attn, 0.70 at gated and 0.64 at x_out; the embeddings and the heads stayed below 0.52.  The 2B and STT cases stayed
below 0.83 at embed (the rule; bit-exact to the bf16 sum), 0.58 at k, 0.74 at v, 0.57 at attn_out, 0.51 at x_attn, 0.59 at
gated, 0.52 at x_out, 0.48 at the heads and 0.65 at the extra heads.

Left out on purpose: 8-bit KV rings (their attention has its own gate, tests/test_gpu_zv_kv_q8.py, and the ring entry is not
a bf16 value the rule could hold), sampling (the samplers are gated by the depformer reference test) and batches past 256
(streaming_begin refuses them).
"""
import dataclasses
import json
import pathlib
import time

import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import MOSHI_7B, LMConfig
from moshi_b200.synth import tiled_lm_state_dict
from tests.util import (device_rope_freqs, extra_heads_ratios, temporal_embed_bf16, temporal_heads_ref64, temporal_layer_ref64,
                        tm_layer_checkpoints, tm_row_ratios)

pytestmark = pytest.mark.gpu

MEMBER = LMConfig.from_dict({**MOSHI_7B.to_reference_kwargs(), "num_layers": 4, "depformer_num_layers": 2})
MEMBER_Q = LMConfig.from_dict({**MOSHI_7B.to_reference_kwargs(), "num_layers": 4, "depformer_num_layers": 2, "quantize": True})
# the 2B model (dim 2560, 20 heads, ffn 7040, 24 layers, n_q 32, dep_q 16, text_card 48000, RoPE period 1e5); its LUT
# conditioner is left out, the cond cases write condition_sum directly
_2B = json.loads((pathlib.Path(__file__).parent / "golden" / "moshi_dev_2b.json").read_text())
TWO_B = LMConfig.from_dict({k: v for k, v in _2B.items() if k not in ("conditioners", "fuser")})
TWO_B_MEMBER = dataclasses.replace(TWO_B, num_layers=4, depformer_num_layers=2)
TWO_B_Q = dataclasses.replace(TWO_B_MEMBER, quantize=True)
# an STT geometry at the width of the 1B models: no depformer, every one of the 32 audio streams from the user, four extra
# heads of six outputs (the shapes the kernels tile by, not a pinned checkpoint config)
STT = LMConfig(dim=2048, num_heads=16, num_layers=4, n_q=32, dep_q=0, text_card=8000, delays=[0] * 33, extra_heads_num_heads=4,
               extra_heads_dim=6)

# (id, model, batches, options): fill = first position (rows add their index mod 13 unless "same_pos"), cap = kv_capacity
CASES = [
    ("7b-B38", "7b", (38,), dict(fill=250, cap=320, steps=2)),
    ("7b-wrap", "7b", (3,), dict(fill=2998, steps=4, same_pos=True)),
    ("member-bf16", "member", (1, 2, 3, 4, 17, 32, 33, 64, 65, 128, 129, 200, 256), dict(fill=200, cap=256, steps=2)),
    ("member-gemv4", "member", (3, 4), dict(fill=200, cap=256, steps=2, gemv_rows=4)),
    ("member-int8", "member_q", (1, 3, 32, 33, 64, 65, 128, 129, 256), dict(fill=200, cap=256, steps=2)),
    ("member-cfg", "member", (20, 65), dict(fill=200, cap=256, steps=2, cfg=3.0, pause=1)),
    ("member-cond", "member", (33,), dict(fill=200, cap=256, steps=2, cond=True)),
    ("member-paged", "member", (38,), dict(fill=200, steps=2, paged=True)),
    ("2b-member-bf16", "2b_member", (1, 2, 3, 4, 17, 32, 33, 64, 65, 128, 129, 200, 256), dict(fill=200, cap=256, steps=2)),
    ("2b-gemv4", "2b_member", (3, 4), dict(fill=200, cap=256, steps=2, gemv_rows=4)),
    ("2b-member-int8", "2b_q", (1, 3, 32, 33, 64, 65, 128, 129, 256), dict(fill=200, cap=256, steps=2)),
    ("2b-cfg-cond", "2b_member", (20, 65), dict(fill=200, cap=256, steps=2, cfg=3.0, pause=1, cond=True)),
    ("2b-paged", "2b_member", (38,), dict(fill=200, steps=2, paged=True)),
    ("2b-B38", "2b", (38,), dict(fill=250, cap=320, steps=2)),
    # an hour at 12.5 Hz: the ring has wrapped 15 times and RoPE at period 1e5 turns far from position 0
    ("2b-hour", "2b", (3,), dict(fill=44998, steps=4, same_pos=True)),
    ("stt", "stt", (1, 2, 3, 4, 33, 64, 65, 129, 256), dict(fill=200, cap=256, steps=2)),
]

_models: dict = {}


def _model(name: str):
    from moshi_b200.models import LMModel
    if name not in _models:
        _models.clear()
        torch.cuda.empty_cache()
        cfg = {"7b": MOSHI_7B, "member": MEMBER, "member_q": MEMBER_Q, "2b": TWO_B, "2b_member": TWO_B_MEMBER, "2b_q": TWO_B_Q,
               "stt": STT}[name]
        sd = tiled_lm_state_dict(cfg, seed=17)
        _models[name] = (cfg, sd, LMModel(cfg, sd, device="cuda"))
    return _models[name]


def _entries(gen) -> dict:
    return {n: (dt, shape, nb) for n, dt, shape, nb in gen._state_entries()}


def _read(gen, ent: dict, name: str) -> torch.Tensor:
    return gen._read_state(name, *ent[name])


def _start(gen, cfg, B: int, opt: dict, seed: int):
    """Writes the session state both runs of a case start from: per-row positions, a token ring of real tokens, rings of
    N(0, 1) history (regenerated from seeded CUDA generators), the condition sum and the exec mask."""
    MB = gen._model_batch
    ent = _entries(gen)
    jit = torch.zeros(MB, dtype=torch.int64) if opt.get("same_pos") else (torch.arange(MB) % B) % 13
    pos = opt["fill"] + jit
    gen._write_state("model.offset", pos)
    gen._write_state("offsets", pos[:B].clone())
    _lib.check(gen._lib.b200_lm_set_offset_cpu(gen._h, int(opt["fill"])))
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt, shape, _ = ent["cache"]
    gen._write_state("cache", torch.randint(0, 2048, shape, generator=g, device="cuda"))
    for l in range(cfg.num_layers):
        for kv in "kv":
            dt, shape, _ = ent[f"layers.{l}.{kv}"]
            gen._write_state(f"layers.{l}.{kv}", torch.randn(shape, generator=g, device="cuda").to(dt))
    cond = None
    if opt.get("cond"):
        cond = (0.5 * torch.randn(MB, cfg.dim, generator=g, device="cuda")).bfloat16()
        _lib.check(gen._lib.b200_lm_set_condition_sum(gen._h, _lib.ptr(cond), MB))
    mask = torch.ones(B, dtype=torch.bool)
    if "pause" in opt:
        mask[opt["pause"]] = False
        gen.set_exec_mask(mask)
    return ent, cond, mask


def _gen(lm, cfg, B: int, opt: dict):
    from moshi_b200.models import LMGen
    c = opt.get("cfg", 1.0)
    gen = LMGen(lm, use_sampling=False, cfg_coef=c, cfg_is_no_text=c != 1.0)
    if opt.get("paged"):
        pages = -(-(opt["fill"] + 13 + opt["steps"]) // 64)
        gen.kv_pool_frames = (2 if c != 1.0 else 1) * B * pages * 64 + 256
    else:
        gen.kv_capacity = opt.get("cap")
    return gen


def _step(gen, cfg, codes: torch.Tensor):
    """One step; the extra heads' probabilities [n, MB, E] as step_with_extra_heads returns them (None without)."""
    if not cfg.extra_heads_num_heads:
        gen.step(codes)
        return None
    _, heads = gen.step_with_extra_heads(codes)
    return torch.stack([h[:, 0] for h in heads])


def _outputs(gen, cfg, MB: int, B: int, extra) -> dict:
    out = {"transformer_out": gen.read_buffer("transformer_out", torch.bfloat16, (MB, cfg.dim)),
           "text_logits": gen.read_buffer("model_text_logits", torch.bfloat16, (MB, cfg.text_card)),
           "text_token": gen.read_buffer("text_token", torch.int64, (B,))}
    if cfg.dep_q > 0:
        out["dep_in"] = gen.read_buffer("dep_in", torch.bfloat16, (MB, cfg.dep_q, cfg.depformer_dim))
        out["audio_tokens"] = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B))
    if extra is not None:
        out["extra_heads"] = extra
    return out


def _exact_ratios(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    bad = got.reshape(got.shape[0], -1) != want.to(got.device).bfloat16().reshape(got.shape[0], -1)
    return bad.any(1).double() * 1e9


@torch.no_grad()
def _run(lm, cfg, sd, B: int, opt: dict, seed: int, res: dict) -> None:
    freqs = device_rope_freqs(cfg.dim // cfg.num_heads, cfg.max_period)
    g = torch.Generator().manual_seed(seed)
    codes = [torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g) for _ in range(opt["steps"])]
    H, D, L = cfg.num_heads, cfg.dim // cfg.num_heads, cfg.num_layers
    kept = []
    gen = _gen(lm, cfg, B, opt)
    with gen.streaming(B):
        MB = gen._model_batch
        ent, cond, mask = _start(gen, cfg, B, opt, seed)
        ex = mask.repeat(MB // B).cuda()
        _lib.check(gen._lib.b200_lm_set_taps(gen._h, 1))
        ar = torch.arange(MB, device="cuda")
        for s in range(opt["steps"]):
            pos = _read(gen, ent, "model.offset")
            paused = {}
            if not bool(ex.all()):
                for l in range(L):
                    for kv in "kv":
                        r = _read(gen, ent, f"layers.{l}.{kv}")
                        paused[(l, kv)] = r[ar, :, pos % r.shape[2]][~ex].clone()
            extra = _step(gen, cfg, codes[s].cuda())
            pos_after = _read(gen, ent, "model.offset")
            if not torch.equal(pos_after, torch.where(ex, pos + 1, pos)):
                res["fail"].append(f"B={B} step {s}: positions {pos.tolist()} -> {pos_after.tolist()}")
            tok = gen.read_buffer("input_tokens", torch.int64, (MB, cfg.n_q + 1))
            x_in = gen.read_buffer("temporal.embed", torch.bfloat16, (MB, cfg.dim))
            # the same chain of bf16 adds as the reference, in its order: bit for bit
            checks = [("embed", None, x_in, temporal_embed_bf16(sd, tok, cond), None)]
            slots = []
            for l in range(L):
                t = {k: gen.read_buffer(f"temporal.layers.{l}.{k}", torch.bfloat16, (MB, n))
                     for k, n in (("attn_out", cfg.dim), ("x_attn", cfg.dim), ("gated", cfg.ffn_hidden), ("x_out", cfg.dim))}
                kr, vr = _read(gen, ent, f"layers.{l}.k"), _read(gen, ent, f"layers.{l}.v")
                cap = kr.shape[2]
                t["k"], t["v"] = kr[ar, :, pos % cap], vr[ar, :, pos % cap]
                slots.append((t["k"].clone(), t["v"].clone()))
                for kv, ring in (("k", kr), ("v", vr)):
                    if (l, kv) in paused and not torch.equal(ring[ar, :, pos % cap][~ex], paused[(l, kv)]):
                        res["fail"].append(f"B={B} step {s} layer {l}: a paused row's {kv} ring slot changed")
                want = temporal_layer_ref64(sd, cfg, l, x_in, t["attn_out"], t["x_attn"], t["gated"], (kr, vr), pos, ex,
                                            rope_freqs=freqs)
                del kr, vr
                checks += [(kind, l, gk, wk, sc) for kind, gk, wk, sc in tm_layer_checkpoints(want, t, ex)]
                x_in = t["x_out"]
                for kind, l_, gk, wk, sc in checks:
                    _judge(res, cfg, B, s, kind, l_, gk, wk, sc)
                checks = []
            out = _outputs(gen, cfg, MB, B, extra)
            heads = temporal_heads_ref64(sd, cfg, x_in, out["transformer_out"])
            for kind in heads:
                _judge(res, cfg, B, s, kind, None, out[kind], heads[kind], None)
            kept.append((slots, out))
    # the same steps from a fresh start, taps off, graph on: bit for bit
    gen = _gen(lm, cfg, B, opt)
    with gen.streaming(B):
        ent, _, _ = _start(gen, cfg, B, opt, seed)
        for s in range(opt["steps"]):
            pos = _read(gen, ent, "model.offset")
            extra = _step(gen, cfg, codes[s].cuda())
            slots, out = kept[s]
            for l in range(L):
                for i, kv in enumerate("kv"):
                    r = _read(gen, ent, f"layers.{l}.{kv}")
                    if not torch.equal(r[ar, :, pos % r.shape[2]], slots[l][i]):
                        res["bitwise"].append(f"B={B} step {s} layer {l} ring {kv}")
            for k, v in _outputs(gen, cfg, gen._model_batch, B, extra).items():
                if not torch.equal(v, out[k]):
                    res["bitwise"].append(f"B={B} step {s} {k}")


def _judge(res: dict, cfg, B: int, s: int, kind: str, layer, got, want, scale) -> None:
    if (cfg.quantize and kind in ("x_attn", "x_out")) or kind == "embed":
        r = _exact_ratios(got, want)
    elif kind == "extra_heads":         # per (head, row): [n, MB] -> the worst head of each row
        r = extra_heads_ratios(got, want).amax(0)
    else:
        r = tm_row_ratios(got, want, kind, scale)
    res["worst"][kind] = max(res["worst"].get(kind, 0.0), float(r.max()))
    if bool((r > 1).any()):
        rows = (r > 1).nonzero().flatten().tolist()
        where = f"layer {layer} " if layer is not None else ""
        res["fail"].append(f"B={B} step {s} {where}{kind}: rows {rows[:8]}{' ...' if len(rows) > 8 else ''} of {r.numel()}, "
                           f"worst ratio {float(r.max()):.3g}")


@pytest.mark.parametrize("case,model,batches,opt", CASES, ids=[c[0] for c in CASES])
def test_temporal_layers_match_fp64_reference(case, model, batches, opt):
    cfg, sd, lm = _model(model)
    t0 = time.time()
    before = _lib.lib().b200_op_set_gemv_max_rows(opt["gemv_rows"]) if "gemv_rows" in opt else None
    failures, bitwise = [], []
    try:
        for B in batches:
            res = dict(worst={}, fail=[], bitwise=[])
            _run(lm, cfg, sd, B, opt, seed=1000 + B, res=res)
            w = res["worst"]
            print(f"\n{case} B={B}: worst ratio " + ", ".join(f"{k} {v:.3f}" for k, v in w.items()) +
                  f"; taps off, graph on: {'bit-identical' if not res['bitwise'] else 'DIFFERS ' + str(res['bitwise'][:4])}")
            failures += [f"{case} " + f for f in res["fail"][:1]]
            bitwise += [f"{case} " + f for f in res["bitwise"][:4]]
    finally:
        if before is not None:
            _lib.lib().b200_op_set_gemv_max_rows(before)
    print(f"{case}: {time.time() - t0:.1f} s")
    assert not failures, "first failing checkpoint:\n" + "\n".join(failures)
    assert not bitwise, "taps off and graph on differ from the tapped steps:\n" + "\n".join(bitwise)


@pytest.mark.parametrize("B", [1, 38])
def test_taps_off_launch_the_same_kernels(B):
    """The taps add copies, never kernels: a step launches as many kernels with the taps off as with them on, before and
    after them, eager and as a captured graph."""
    from moshi_b200.models import LMGen
    cfg, sd, lm = _model("member")
    lib = _lib.lib()
    codes = torch.zeros(B, cfg.n_q - cfg.dep_q, 1, dtype=torch.int64, device="cuda")
    for graph in (False, True):
        gen = LMGen(lm, use_sampling=False)
        gen.use_graph = graph
        gen.kv_capacity = 64
        counts = []
        with gen.streaming(B):
            for taps in (0, 1, 0):
                _lib.check(gen._lib.b200_lm_set_taps(gen._h, taps))
                gen.step(codes)                              # captures the graph (its launch is counted like a replay)
                torch.cuda.synchronize()
                n0 = lib.b200_launch_count()
                gen.step(codes)
                torch.cuda.synchronize()
                counts.append(lib.b200_launch_count() - n0)
        print(f"\nB={B} {'graph' if graph else 'eager'}: kernels per step with taps off, on, off: {counts}")
        assert counts[0] == counts[1] == counts[2], counts
