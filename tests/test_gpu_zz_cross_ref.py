"""GPU: every layer of a cross-attention LM (the TTS models' temporal transformer) against the fp64 reference, teacher-forced on
per-layer taps, at a TTS-like geometry and serving batch, for every linear schedule of the cross block; the condition memory's
fill against fp64; then the same steps without taps, bit for bit; and the edges of cross_attn_step_kernel the handle's
shapes do not reach.

The member: dim 2048, 16 heads, ffn 5632, three temporal layers with cross-attention, a tensor conditioner of dim 512 fused
by ``cross`` with the positional embedding, dep_q 4 and one depformer layer, synthetic tiled weights; condition memories of
T = 125 and 625 keys.  Batches 1-2 put the cross query and output linears (dim x dim) on the GEMV, 3-32 on swap-AB
stream-K, 33-128 on the non-swapped kernel and 129-256 on that kernel as two 128-row blocks; "gemv4" raises the GEMV's row
limit to 4.  A 7B-geometry member (dim 4096, 32 heads) runs B = 3 and 38 for H = 32 and K = 4096 in the cross linears.  The
rings hold random history a few hundred frames in, per-row positions; the CFG case gives each half of the 2B model rows its
own memory and pauses one row; the paged case runs the self-attention rings from the page pool.

Per case and batch:

* memory fill: after streaming_begin every row's k_cross / v_cross against cross_memory_ref64 of its fused condition; then
  set_condition_cross on an out-of-order, non-contiguous subset of the model rows ([200, 3, 129] at 256 rows) with new
  conditions: those rows against the reference, every other row bit-identical to before;
* per step with b200_lm_set_taps on, under the rule of tests/util.py (constants calibrated by tests/test_cross_ref_cpu.py):
  the embeddings, then every layer's new k and v, attn_out, x_attn, cross_out, x_cross, gated and x_out (the MLP judged on
  the x_cross tap), then transformer_out, the text logits and dep_in; the steps leave every row's memory bit-identical;
* the same steps from a fresh start, with the same memory, taps off and the step graph on: ring entries, transformer_out,
  text logits, dep_in and tokens bit-identical.  The cross block puts layernorm_kernel and cross_attn_step_kernel between
  the PDL-launched GEMMs, and its two taps change which kernels are adjacent.

A failure names the first failing (step, layer, checkpoint, rows).

On one H100 80GB HBM3 (power limit 700 W) the whole file takes about 50 s, building the models included.  The worst ratios it
met (1 = at the tolerance) were 0.48 at kx / vx, 0.46 at cross_out and 0.49 at x_cross; at the other checkpoints 0.79 at
k, 0.66 at attn_out, 0.64 at x_out, 0.52 at gated, the rest below 0.5.

Left out on purpose: int8 linears (refused with cross-attention), 8-bit KV rings (tests/test_gpu_zv_kv_q8.py) and sampling
(gated by the depformer and noise tests).
"""
import ctypes as C
import time

import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import LMConfig
from moshi_b200.synth import tiled_lm_state_dict
from tests.util import (cptr, cross_memory_ref64, device_rope_freqs, err_ratios, temporal_embed_ref64, temporal_heads_ref64,
                        temporal_layer_ref64, tm_layer_checkpoints, tm_row_ratios)

pytestmark = pytest.mark.gpu

COND = {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 512}}}
FUSER = {"cross": ["speaker_wavs"], "cross_attention_pos_emb": True, "cross_attention_pos_emb_scale": 0.5}
_SMALL = dict(text_card=8000, n_q=8, dep_q=4, delays=[0] + [1] * 8, depformer_num_layers=1, cross_attention=True,
              conditioners=COND, fuser=FUSER)
TTS = LMConfig.from_dict({"dim": 2048, "num_heads": 16, "num_layers": 3, **_SMALL})
TTS_7B = LMConfig.from_dict({"num_layers": 2, **_SMALL})

ALL_B = (1, 2, 3, 4, 17, 32, 33, 64, 65, 128, 129, 200, 256)
# (id, model, batches, options): T = condition keys, fill = first position (rows add their index mod 13), cap = kv_capacity
CASES = [
    ("tts-T125", "tts", ALL_B, dict(T=125, fill=200, cap=256, steps=2)),
    ("tts-T625", "tts", ALL_B, dict(T=625, fill=200, cap=256, steps=2)),
    ("tts-gemv4", "tts", (3, 4), dict(T=125, fill=200, cap=256, steps=2, gemv_rows=4)),
    ("tts-cfg", "tts", (20, 65), dict(T=125, fill=200, cap=256, steps=2, cfg=3.0, pause=1)),
    ("tts-paged", "tts", (38,), dict(T=125, fill=200, steps=2, paged=True)),
    ("7b-cross", "7b", (3, 38), dict(T=125, fill=250, cap=320, steps=2)),
]

_models: dict = {}


def _model(name: str):
    from moshi_b200.models import LMModel
    if name not in _models:
        _models.clear()
        torch.cuda.empty_cache()
        cfg = {"tts": TTS, "7b": TTS_7B}[name]
        sd = tiled_lm_state_dict(cfg, seed=19)
        _models[name] = (cfg, sd, LMModel(cfg, sd, device="cuda"))
    return _models[name]


def _conditions(lm, n: int, T: int, seed: int):
    """Condition tensors of n random voices [1, T, 512] and their fused condition (fuser.get_cross) [n, T, dim] bf16."""
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    g = torch.Generator().manual_seed(seed)
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(torch.randn(1, T, 512, generator=g))})
             for _ in range(n)]
    ct = lm.condition_provider(lm.condition_provider.prepare(attrs))
    return ct, lm.fuser.get_cross(ct).to(device="cuda", dtype=torch.bfloat16).contiguous()


def _subset(MB: int) -> list[int]:
    """Out of order and not contiguous: [200, 3, 129] at 256 model rows."""
    return list(dict.fromkeys([200 % MB, 3 % MB, 129 % MB]))


def _entries(gen) -> dict:
    return {n: (dt, shape, nb) for n, dt, shape, nb in gen._state_entries()}


def _read(gen, ent: dict, name: str) -> torch.Tensor:
    return gen._read_state(name, *ent[name])


def _gen(lm, B: int, opt: dict, ct):
    from moshi_b200.models import LMGen
    c = opt.get("cfg", 1.0)
    gen = LMGen(lm, use_sampling=False, cfg_coef=c, condition_tensors=ct)
    if opt.get("paged"):
        pages = -(-(opt["fill"] + 13 + opt["steps"]) // 64)
        gen.kv_pool_frames = (2 if c != 1.0 else 1) * B * pages * 64 + 256
    else:
        gen.kv_capacity = opt.get("cap")
    return gen


def _start(gen, cfg, B: int, opt: dict, seed: int):
    """Writes the session state both runs of a case start from: per-row positions, a token ring of real tokens, rings of
    N(0, 1) history (from seeded CUDA generators) and the exec mask."""
    MB = gen._model_batch
    ent = _entries(gen)
    pos = opt["fill"] + (torch.arange(MB) % B) % 13
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
    mask = torch.ones(B, dtype=torch.bool)
    if "pause" in opt:
        mask[opt["pause"]] = False
        gen.set_exec_mask(mask)
    return ent, mask


def _memory(gen, ent: dict, cfg) -> list[tuple[torch.Tensor, torch.Tensor]]:
    return [(_read(gen, ent, f"layers.{l}.k_cross"), _read(gen, ent, f"layers.{l}.v_cross")) for l in range(cfg.num_layers)]


def _judge_memory(res: dict, sd: dict, cfg, mem, src: torch.Tensor, rows: list[int] | None, what: str) -> None:
    """The memory of model rows ``rows`` (None: all) against cross_memory_ref64 of their fused condition ``src``."""
    idx = torch.arange(src.shape[0], device="cuda") if rows is None else torch.tensor(rows, device="cuda")
    for l, (kx, vx) in enumerate(mem):
        for r0, k, v in cross_memory_ref64(sd, cfg, l, src, rows=16):
            sel = idx[r0:r0 + k.shape[0]]
            for kind, got, want in (("kx", kx[sel], k), ("vx", vx[sel], v)):
                r = tm_row_ratios(got, want, kind)
                res["worst"][kind] = max(res["worst"].get(kind, 0.0), float(r.max()))
                if bool((r > 1).any()):
                    bad = sel[(r > 1).nonzero().flatten()].tolist()
                    res["fail"].append(f"{what}: layer {l} {kind}: model rows {bad[:8]}, worst ratio {float(r.max()):.3g}")


def _fill(gen, lm, cfg, sd, B: int, opt: dict, seed: int, res: dict | None):
    """The memory of a fresh session, then a new condition for an out-of-order subset of rows; judged when ``res`` is given.
    Returns the memory after both."""
    MB = gen._model_batch
    ent = _entries(gen)
    rows = _subset(MB)
    _, src_new = _conditions(lm, len(rows), opt["T"], seed + 1)
    before = _memory(gen, ent, cfg) if res is not None else None
    gen.set_condition_cross(src_new, rows)
    after = _memory(gen, ent, cfg)
    if res is not None:
        _judge_memory(res, sd, cfg, before, res["src"], None, f"B={B} fill at streaming_begin")
        _judge_memory(res, sd, cfg, after, src_new, rows, f"B={B} set_condition_cross {rows}")
        others = torch.ones(MB, dtype=torch.bool, device="cuda")
        others[rows] = False
        for l in range(cfg.num_layers):
            for i, kv in enumerate("kv"):
                if not torch.equal(after[l][i][others], before[l][i][others]):
                    res["fail"].append(f"B={B} set_condition_cross {rows}: layer {l} {kv}_cross of another row changed")
    return after


def _outputs(gen, cfg, MB: int, B: int) -> dict:
    return {"transformer_out": gen.read_buffer("transformer_out", torch.bfloat16, (MB, cfg.dim)),
            "text_logits": gen.read_buffer("model_text_logits", torch.bfloat16, (MB, cfg.text_card)),
            "dep_in": gen.read_buffer("dep_in", torch.bfloat16, (MB, cfg.dep_q, cfg.depformer_dim)),
            "text_token": gen.read_buffer("text_token", torch.int64, (B,)),
            "audio_tokens": gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B))}


def _judge(res: dict, B: int, s: int, kind: str, layer, got, want, scale) -> None:
    r = tm_row_ratios(got, want, kind, scale)
    res["worst"][kind] = max(res["worst"].get(kind, 0.0), float(r.max()))
    if bool((r > 1).any()):
        rows = (r > 1).nonzero().flatten().tolist()
        where = f"layer {layer} " if layer is not None else ""
        res["fail"].append(f"B={B} step {s} {where}{kind}: rows {rows[:8]}{' ...' if len(rows) > 8 else ''} of {r.numel()}, "
                           f"worst ratio {float(r.max()):.3g}")


@torch.no_grad()
def _run(lm, cfg, sd, B: int, opt: dict, seed: int, res: dict) -> None:
    freqs = device_rope_freqs(cfg.dim // cfg.num_heads, cfg.max_period)
    g = torch.Generator().manual_seed(seed)
    codes = [torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g) for _ in range(opt["steps"])]
    MB = B * (2 if opt.get("cfg", 1.0) != 1.0 else 1)
    ct, res["src"] = _conditions(lm, MB, opt["T"], seed)
    L = cfg.num_layers
    kept = []
    gen = _gen(lm, B, opt, ct)
    with gen.streaming(B):
        mem = _fill(gen, lm, cfg, sd, B, opt, seed, res)
        ent, mask = _start(gen, cfg, B, opt, seed)
        ex = mask.repeat(MB // B).cuda()
        _lib.check(gen._lib.b200_lm_set_taps(gen._h, 1))
        ar = torch.arange(MB, device="cuda")
        for s in range(opt["steps"]):
            pos = _read(gen, ent, "model.offset")
            gen.step(codes[s].cuda())
            pos_after = _read(gen, ent, "model.offset")
            if not torch.equal(pos_after, torch.where(ex, pos + 1, pos)):
                res["fail"].append(f"B={B} step {s}: positions {pos.tolist()} -> {pos_after.tolist()}")
            tok = gen.read_buffer("input_tokens", torch.int64, (MB, cfg.n_q + 1))
            x_in = gen.read_buffer("temporal.embed", torch.bfloat16, (MB, cfg.dim))
            _judge(res, B, s, "embed", None, x_in, temporal_embed_ref64(sd, cfg, tok), None)
            slots = []
            for l in range(L):
                t = {k: gen.read_buffer(f"temporal.layers.{l}.{k}", torch.bfloat16, (MB, n))
                     for k, n in (("attn_out", cfg.dim), ("x_attn", cfg.dim), ("cross_out", cfg.dim), ("x_cross", cfg.dim),
                                  ("gated", cfg.ffn_hidden), ("x_out", cfg.dim))}
                kr, vr = _read(gen, ent, f"layers.{l}.k"), _read(gen, ent, f"layers.{l}.v")
                cap = kr.shape[2]
                t["k"], t["v"] = kr[ar, :, pos % cap], vr[ar, :, pos % cap]
                slots.append((t["k"].clone(), t["v"].clone()))
                cross = dict(cross_out=t["cross_out"], x_cross=t["x_cross"], kx=mem[l][0], vx=mem[l][1])
                want = temporal_layer_ref64(sd, cfg, l, x_in, t["attn_out"], t["x_attn"], t["gated"], (kr, vr), pos, ex,
                                            rope_freqs=freqs, cross=cross)
                del kr, vr
                for kind, gk, wk, sc in tm_layer_checkpoints(want, t, ex):
                    _judge(res, B, s, kind, l, gk, wk, sc)
                x_in = t["x_out"]
            out = _outputs(gen, cfg, MB, B)
            heads = temporal_heads_ref64(sd, cfg, x_in, out["transformer_out"])
            for kind in ("transformer_out", "text_logits", "dep_in"):
                _judge(res, B, s, kind, None, out[kind], heads[kind], None)
            kept.append((slots, out))
        for l, (kx, vx) in enumerate(_memory(gen, ent, cfg)):
            if not (torch.equal(kx, mem[l][0]) and torch.equal(vx, mem[l][1])):
                res["fail"].append(f"B={B}: the steps changed layer {l}'s condition memory")
    del mem
    # the same steps from a fresh start with the same memory, taps off, graph on: bit for bit
    gen = _gen(lm, B, opt, ct)
    with gen.streaming(B):
        _fill(gen, lm, cfg, sd, B, opt, seed, None)
        ent, _ = _start(gen, cfg, B, opt, seed)
        for s in range(opt["steps"]):
            pos = _read(gen, ent, "model.offset")
            gen.step(codes[s].cuda())
            slots, out = kept[s]
            for l in range(L):
                for i, kv in enumerate("kv"):
                    r = _read(gen, ent, f"layers.{l}.{kv}")
                    if not torch.equal(r[ar, :, pos % r.shape[2]], slots[l][i]):
                        res["bitwise"].append(f"B={B} step {s} layer {l} ring {kv}")
            for k, v in _outputs(gen, cfg, MB, B).items():
                if not torch.equal(v, out[k]):
                    res["bitwise"].append(f"B={B} step {s} {k}")


@pytest.mark.parametrize("case,model,batches,opt", CASES, ids=[c[0] for c in CASES])
def test_cross_layers_match_fp64_reference(case, model, batches, opt):
    cfg, sd, lm = _model(model)
    t0 = time.time()
    before = _lib.lib().b200_op_set_gemv_max_rows(opt["gemv_rows"]) if "gemv_rows" in opt else None
    failures, bitwise = [], []
    try:
        for B in batches:
            res = dict(worst={}, fail=[], bitwise=[])
            _run(lm, cfg, sd, B, opt, seed=2000 + B + opt["T"], res=res)
            w = res["worst"]
            print(f"\n{case} B={B}: worst ratio " + ", ".join(f"{k} {v:.3f}" for k, v in w.items()) +
                  f"; taps off, graph on: {'bit-identical' if not res['bitwise'] else 'DIFFERS ' + str(res['bitwise'][:4])}")
            failures += [f"{case} " + f for f in res["fail"][:1]]
            bitwise += [f"{case} " + f for f in res["bitwise"][:4]]
            torch.cuda.empty_cache()
    finally:
        if before is not None:
            _lib.lib().b200_op_set_gemv_max_rows(before)
    print(f"{case}: {time.time() - t0:.1f} s")
    assert not failures, "first failing checkpoint:\n" + "\n".join(failures)
    assert not bitwise, "taps off and graph on differ from the tapped steps:\n" + "\n".join(bitwise)


# ---- cross_attn_step_kernel at its edges ---------------------------------------------------------------------------------
def _cross_attn(q, k, v, B: int, H: int, T: int, nsplit: int) -> torch.Tensor:
    out = torch.empty(B, H * 128, dtype=torch.bfloat16, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib().b200_op_cross_attn_step(cptr(q), cptr(k), cptr(v), cptr(out), B, H, T, nsplit, s))
    torch.cuda.synchronize()
    return out.view(B, H, 128)


def _attn64(q, k, v, rows: int = 8) -> torch.Tensor:
    """softmax(q . k_t / sqrt(128)) . v_t over all T keys in float64 on the device, a few rows at a time."""
    out = []
    for i in range(0, q.shape[0], rows):
        kk, vv = k[i:i + rows].double(), v[i:i + rows].double()
        p = torch.softmax(torch.einsum("bhd,bhtd->bht", q[i:i + rows].double(), kk) * 128 ** -0.5, dim=-1)
        out.append(torch.einsum("bht,bhtd->bhd", p, vv))
        del kk, vv, p
    return torch.cat(out)


@pytest.mark.parametrize("B,H,T,nsplit", [(3, 2, 5, 4), (2, 16, 65, 16), (5, 16, 1, 4)])
def test_cross_attn_splits_without_keys(B, H, T, nsplit):
    """An explicit split count that leaves the last splits with no key (T = 5 over 4 splits of 2: the fourth starts at 6;
    T = 65 over 16 splits of 5: splits 13-15 are empty): they must merge as nothing."""
    g = torch.Generator(device="cuda").manual_seed(T * 100 + nsplit)
    q = torch.randn(B, H, 128, generator=g, device="cuda").bfloat16()
    k = torch.randn(B, H, T, 128, generator=g, device="cuda").bfloat16()
    v = torch.randn(B, H, T, 128, generator=g, device="cuda").bfloat16()
    k[:, :, T - 1] = q                       # a needle at the last key, in the last split that has one
    ratio = float(err_ratios(_cross_attn(q, k, v, B, H, T, nsplit), _attn64(q, k, v)).max())
    print(f"cross attn B={B} H={H} T={T} nsplit={nsplit}: worst err / tolerance {ratio:.3f}")
    assert ratio <= 1.0


def test_cross_attn_zero_memory_rows():
    """Memory rows of zeros (a condition whose positions are all masked and project to zero): uniform weights over zero
    values give exact zeros; a row zero from half its keys on attends to them with score 0."""
    B, H, T = 4, 16, 125
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(B, H, 128, generator=g, device="cuda").bfloat16()
    k = torch.randn(B, H, T, 128, generator=g, device="cuda").bfloat16()
    v = torch.randn(B, H, T, 128, generator=g, device="cuda").bfloat16()
    k[0], v[0] = 0, 0
    k[2, :, T // 2:], v[2, :, T // 2:] = 0, 0
    for nsplit in (0, 1, 3):
        got = _cross_attn(q, k, v, B, H, T, nsplit)
        assert bool((got[0] == 0).all()), nsplit
        ratio = float(err_ratios(got[1:], _attn64(q, k, v)[1:]).max())
        print(f"zero memory rows, nsplit={nsplit}: worst err / tolerance {ratio:.3f}")
        assert ratio <= 1.0


def test_cross_attn_memory_past_2_31_elements():
    """B = 256, H = 16, T = 4200: k and v hold 2.2 G elements each (8.8 GB together), so the (row, head) offsets of the last
    rows pass 2^31 and a 32-bit index anywhere in the kernel reads the wrong keys.  A needle key (the query itself) at the
    first, last or a middle key of every row."""
    B, H, T = 256, 16, 4200
    assert B * H * T * 128 > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(31)
    q = torch.randn(B, H, 128, generator=g, device="cuda").bfloat16()
    k = torch.randn(B, H, T, 128, generator=g, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(B, H, T, 128, generator=g, device="cuda", dtype=torch.bfloat16)
    for b in range(B):
        k[b, :, [0, T - 1, T // 2][b % 3]] = q[b]
    try:
        want = _attn64(q, k, v)
        high = (torch.arange(B, device="cuda") * H + H - 1) * T * 128 >= 2 ** 31
        for nsplit in (0, 3):
            r = err_ratios(_cross_attn(q, k, v, B, H, T, nsplit), want).flatten(1).amax(1)
            print(f"cross attn B={B} H={H} T={T} nsplit={nsplit}: worst err / tolerance {float(r.max()):.3f} "
                  f"({float(r[high].max()):.3f} over the {int(high.sum())} rows past 2^31)")
            assert float(r.max()) <= 1.0, (nsplit, (r > 1).nonzero().flatten().tolist()[:8])
    finally:
        del k, v
        torch.cuda.empty_cache()
