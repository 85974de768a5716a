"""CPU: the fp64 reference of the cross-attention block and of the condition memory, and the acceptance rule of
tests/test_gpu_zz_cross_ref.py, at TTS-like layer shapes (dim 2048, 16 heads, ffn 5632, a tensor conditioner of dim 512
fused by ``cross`` with the positional embedding, T = 125 condition keys) with two layers and a 64-slot ring.

``cross_block_ref64`` and ``cross_memory_ref64`` (tests/util.py) restate the block ``x = x + cross_attention(norm_cross(x),
memory)`` and the memory ``k_cross | v_cross = condition . in_projs.0[d:3d]^T`` in float64 with the bf16 model's cast points,
teacher-forced on the implementation's taps (x after the self-attention residual, the cross-attention output, x after the
cross residual, its own memory); ``temporal_layer_ref64`` runs the MLP on the x_cross tap.  Shown here:

* The rule accepts a correct bf16 cross-attention LM: the bf16 oracle (tests/cross_oracle.py, pinned on the reference by
  tests/golden/lm_tiny_cross), whose activations are recorded at the same taps, passes every checkpoint of two steps at B = 4
  and B = 256 (rings of random history at positions 50..69), and its memory passes kx / vx.  Each constant of TM_C is about
  twice what it needs or more (the test prints both; tests/util.py says which were set from the GPU handle).
* The rule rejects layers with a bug: each mutant below computes a subtly wrong cross block, memory or MLP input (at layer 1,
  step 1 of B = 256), and the checkpoint named beside it must reject it in every row the bug touches.

Not claimed: ulp-level cast-point mutants inside the cross block (a missing bf16 round of the LayerNorm output, of q or of
the attention output).  Such a bug moves a value by at most half a bf16 ulp, which the rule's 2^-7 relative term admits by
design.  Nor is a bug that only reorders the T keys of a row together with their values caught: attention over all keys
without a mask or positions does not depend on their order (the fuser's positional embedding is inside the keys).
"""
import contextlib
import math

import pytest
import torch

from moshi_b200.conditioners import ConditionAttributes, TensorCondition, build_conditioning
from moshi_b200.config import LMConfig
from moshi_b200.synth import iter_synth_lm_tensors
from oracle import transformer as tr
from oracle.lm import LMSpec
from tests.cross_oracle import CrossLMOracle, cross_kv
from tests.util import (TM_C, TM_REL, cross_memory_ref64, temporal_embed_ref64, temporal_heads_ref64, temporal_layer_ref64,
                        tm_c_needed, tm_layer_checkpoints, tm_row_ratios)

COND = {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 512}}}
FUSER = {"cross": ["speaker_wavs"], "cross_attention_pos_emb": True, "cross_attention_pos_emb_scale": 0.5}
CFG = LMConfig(dim=2048, num_heads=16, num_layers=2, context=64, depformer_num_layers=1, cross_attention=True,
               conditioners=COND, fuser=FUSER)
T = 125
STEPS = 2
LAYER, STEP = 1, 1          # where the mutants act
KEEP = ("emb.", "text_emb.", "text_linear.", "out_norm.", "transformer.", "depformer_in.", "condition_provider.")


@pytest.fixture(scope="module")
def sd():
    return {k: v for k, v in iter_synth_lm_tensors(CFG, seed=31) if k.startswith(KEEP)}


def _conditions(sd: dict, B: int, seed: int) -> tuple[torch.Tensor, torch.Tensor]:
    """fuser.get_cross of B random voices [B, T, 512] in bf16, with and without the fuser's positional embedding."""
    g = torch.Generator().manual_seed(seed)
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(torch.randn(1, T, 512, generator=g))})
             for _ in range(B)]
    out = []
    for fuser_cfg in (FUSER, {"cross": FUSER["cross"]}):
        provider, fuser = build_conditioning(COND, fuser_cfg, CFG.dim, sd, "cpu", cross_attention=True)
        out.append(fuser.get_cross(provider(provider.prepare(attrs))).to(torch.bfloat16))
    return out[0], out[1]


@contextlib.contextmanager
def _recording(sd: dict, L: int):
    """Records the inputs of the self-attention and MLP linears and of the norms the oracle runs: log of (key, x, y)."""
    names = {id(sd[f"transformer.layers.{l}.{k}"]): (n, l) for l in range(L)
             for n, k in (("out", "self_attn.out_projs.0.weight"), ("lin_out", "gating.linear_out.weight"))}
    log = []
    lin0, norm0 = tr.linear, tr.apply_norm

    def linear(x, w, quantize=False):
        y = lin0(x, w, quantize)
        if id(w) in names:
            log.append((names[id(w)], x[:, 0], y[:, 0]))
        return y

    def apply_norm(kind, x, sd_, prefix):
        log.append((("norm", prefix), x[:, 0], None))
        return norm0(kind, x, sd_, prefix)

    tr.linear, tr.apply_norm = linear, apply_norm
    try:
        yield log
    finally:
        tr.linear, tr.apply_norm = lin0, norm0


def _oracle_run(sd: dict, B: int, seed: int) -> dict:
    """STEPS oracle steps with history in the rings; per step the taps, rings and heads, and the rows' condition memory."""
    cross, cross_nopos = _conditions(sd, B, seed)
    orc = CrossLMOracle(sd, LMSpec.from_config(CFG), condition_cross=cross, use_sampling=False)
    orc.streaming(B)
    g = torch.Generator().manual_seed(seed)
    st = orc.main_state
    pos = 50 + (torch.arange(B) * 5) % 20
    for ls in st.layers:
        ls.k.copy_(torch.randn(ls.k.shape, generator=g).bfloat16())
        ls.v.copy_(torch.randn(ls.v.shape, generator=g).bfloat16())
        ls.end_offset.copy_(pos)
        ls.offset.copy_(pos)
    st.offsets.copy_(pos)
    steps = []
    L = CFG.num_layers
    for _ in range(STEPS):
        tok = torch.randint(0, CFG.card, (B, CFG.n_q + 1), generator=g)
        tok[::3, 5] = -1
        orc.layer_taps = []
        with _recording(sd, L) as log:
            tout, logits = orc.forward_text(tok[:, :, None])
        norms = {key: x for key, x, _ in log if key[0] == "norm"}
        lins = {key: (x, y) for key, x, y in log if key[0] != "norm"}
        layers = []
        for l in range(L):
            t = {k: v[:, 0] for k, v in orc.layer_taps[l].items()}
            layers.append(dict(x_in=norms[("norm", f"transformer.layers.{l}.norm1")], attn_out=lins[("out", l)][0],
                               x_attn=t["x_attn"], cross_out=t["cross_out"], x_cross=t["x_cross"], gated=lins[("lin_out", l)][0],
                               x_out=t["x_out"], ring=(st.layers[l].k.clone(), st.layers[l].v.clone())))
        tout = tout[:, 0]
        din = torch.stack([tr.linear(tout, sd[f"depformer_in.{k}.weight"]) for k in range(CFG.dep_q)], dim=1)
        steps.append(dict(tokens=tok, pos=pos.clone(), layers=layers, tout=tout, text_logits=logits[:, 0, 0], dep_in=din))
        pos = pos + 1
    return dict(steps=steps, memory=orc.memory, cross=cross, cross_nopos=cross_nopos)


def _checkpoints(sd: dict, run: dict, s: int, mutant: dict | None = None, layers=None):
    """(name, kind, got, want, rms source) of one oracle step against the references, in the order the step computes them.
    Besides temporal_layer_ref64's mutants: "memory": f(k, v) -> the memory the mutant reads; "mlp_x_attn": the MLP reads
    x_attn instead of x_cross."""
    mutant = mutant or {}
    step = run["steps"][s]
    B = step["tokens"].shape[0]
    ex = torch.ones(B, dtype=torch.bool)
    pos = step["pos"]
    ar = torch.arange(B)
    L = step["layers"]
    out = [("embed", "embed", L[0]["x_in"], temporal_embed_ref64(sd, CFG, step["tokens"]), None)] if layers is None else []
    for l in range(len(L)) if layers is None else layers:
        t = L[l]
        kr, vr = t["ring"]
        cap = kr.shape[2]
        kx, vx = run["memory"][l]
        if "memory" in mutant:
            kx, vx = mutant["memory"](kx, vx)
        cross = dict(cross_out=t["cross_out"], x_cross=t["x_attn"] if mutant.get("mlp_x_attn") else t["x_cross"], kx=kx, vx=vx)
        want = temporal_layer_ref64(sd, CFG, l, t["x_in"], t["attn_out"], t["x_attn"], t["gated"], t["ring"], pos, ex, mutant,
                                    cross=cross)
        got = dict(k=kr[ar, :, pos % cap], v=vr[ar, :, pos % cap], attn_out=t["attn_out"], x_attn=t["x_attn"],
                   cross_out=t["cross_out"], x_cross=t["x_cross"], gated=t["gated"], x_out=t["x_out"])
        out += [(f"layer {l} {kind}", kind, g, w, sc) for kind, g, w, sc in tm_layer_checkpoints(want, got, ex)]
    if layers is None:
        heads = temporal_heads_ref64(sd, CFG, L[-1]["x_out"], step["tout"])
        out += [(k, k, step[k] if k != "transformer_out" else step["tout"], heads[k], None)
                for k in ("transformer_out", "text_logits", "dep_in")]
    return out


def _memory_needs(sd: dict, got: tuple[torch.Tensor, torch.Tensor], cross: torch.Tensor, layer: int) -> dict:
    """Per kind "kx" / "vx": the c each row of a memory needs [B] against cross_memory_ref64 of ``cross`` (the rule passes a
    row where this is at most TM_C: tm_c_needed per row, one pass over the 65 M values of a B = 256 memory)."""
    out = {"kx": [], "vx": []}
    for r0, k, v in cross_memory_ref64(sd, CFG, layer, cross, rows=32):
        for kind, g, w in (("kx", got[0], k), ("vx", got[1], v)):
            g = g[r0:r0 + w.shape[0]].double()
            rms = w.pow(2).mean(-1, keepdim=True).sqrt_()
            need = g.sub_(w).abs_().sub_(TM_REL * w.abs()).div_(rms)
            out[kind].append(torch.nan_to_num(need, nan=math.inf).flatten(1).amax(1).clamp(min=0))
    return {kind: torch.cat(r) for kind, r in out.items()}


@pytest.fixture(scope="module")
def runs(sd):
    return {B: _oracle_run(sd, B, seed=B) for B in (4, 256)}


@torch.no_grad()
def test_bf16_oracle_passes_every_checkpoint(sd, runs):
    need, bad = {}, []
    for B, run in runs.items():
        nb = {}
        for l in range(CFG.num_layers):
            for kind, rn in _memory_needs(sd, run["memory"][l], run["cross"], l).items():
                nb[kind] = max(nb.get(kind, 0.0), float(rn.max()))
                if (rn > TM_C[kind]).any():
                    bad.append((B, f"layer {l} {kind}", float(rn.max())))
        for s in range(STEPS):
            for name, kind, g, w, sc in _checkpoints(sd, run, s):
                nb[kind] = max(nb.get(kind, 0.0), tm_c_needed(g, w, sc))
                r = tm_row_ratios(g, w, kind, sc)
                if (r > 1).any():
                    bad.append((B, s, name, float(r.max())))
        print(f"\nB = {B}: c the bf16 oracle needs: " + ", ".join(f"{k} {v:.2e}" for k, v in nb.items()))
        for k, v in nb.items():
            need[k] = max(need.get(k, 0.0), v)
    print("c used: " + ", ".join(f"{k} {TM_C[k]:.2e} ({TM_C[k] / max(need[k], 1e-30):.1f}x)" for k in need))
    assert not bad, bad


# ---- mutants ---------------------------------------------------------------------------------------------------------------
def _kblock(name: str, layer, kb: int = 5):
    """One 64-deep k-block (columns kb*64 .. kb*64+63) of the weight of one linear zeroed."""
    def f(n, ll, fetch):
        w = fetch(n, ll)
        if (n, ll) == (name, layer):
            w = w.clone()
            w[:, kb * 64:(kb + 1) * 64] = 0
        return w
    return {"weight": f}


def _norm_cross(name: str, value: float):
    """norm_cross's weight (ncw) or bias (ncb) of LAYER replaced by a constant: the LayerNorm without it."""
    def f(n, ll, fetch):
        w = fetch(n, ll)
        return torch.full_like(w, value) if (n, ll) == (name, LAYER) else w
    return {"weight": f}


def _shift_one_t(k: torch.Tensor, v: torch.Tensor):
    """Key t of every row holds key t - 1 over the flat (row, t) order of the fill: key 0 the previous row's last key."""
    def sh(x):
        B, H, T_, D = x.shape
        return x.permute(0, 2, 1, 3).reshape(B * T_, H, D).roll(1, 0).view(B, T_, H, D).permute(0, 2, 1, 3)
    return sh(k), sh(v)


ALL = slice(None)
MUTANTS = {
    # name: (mutant, checkpoint that must reject it, rows it touches)
    "one 64-key block of the memory dropped": ({"memory": lambda k, v: (k[:, :, 64:], v[:, :, 64:])}, "cross_out", ALL),
    "another row's memory": ({"memory": lambda k, v: (k.roll(1, 0), v.roll(1, 0))}, "cross_out", ALL),
    "memory shifted by one t": ({"memory": _shift_one_t}, "cross_out", ALL),
    "K and V swapped": ({"memory": lambda k, v: (v, k)}, "cross_out", ALL),
    "LayerNorm without its bias": (_norm_cross("ncb", 0.0), "cross_out", ALL),
    "LayerNorm without its weight": (_norm_cross("ncw", 1.0), "cross_out", ALL),
    "k-block missing: query linear": (_kblock("cq", LAYER), "cross_out", ALL),
    "k-block missing: output linear": (_kblock("co", LAYER), "x_cross", ALL),
    "cross residual dropped": ({"residual": lambda l, w: (l, w) != (LAYER, "cross")}, "x_cross", ALL),
    "MLP fed x_attn instead of x_cross": ({"mlp_x_attn": True}, "gated", ALL),
}


@pytest.mark.parametrize("name", list(MUTANTS))
@torch.no_grad()
def test_mutant_rejected_at_its_checkpoint_in_every_row(sd, runs, name):
    mutant, kind, rows = MUTANTS[name]
    run = runs[256]
    key = f"layer {LAYER} {kind}"
    _, w, s = {n: (g, w, s) for n, _, g, w, s in _checkpoints(sd, run, STEP, layers=[LAYER])}[key]
    got = {n: w for n, _, _, w, _ in _checkpoints(sd, run, STEP, mutant, layers=[LAYER])}[key].bfloat16()
    r = tm_row_ratios(got, w, kind, s)
    print(f"{name}: rejected at {key}, smallest row ratio {float(r[rows].min()):.3g}, "
          f"need {tm_c_needed(got, w, s):.3g} vs c {TM_C[kind]:.3g}")
    assert (r[rows] > 1).all(), (name, r[rows])


@torch.no_grad()
def test_memory_without_the_positional_embedding_is_rejected(sd, runs):
    """The memory filled from the condition without the fuser's positional embedding: kx rejects it in every row."""
    run = runs[256]
    k, v = cross_kv(sd, f"transformer.layers.{LAYER}", run["cross_nopos"], CFG.num_heads)
    need = _memory_needs(sd, (k, v), run["cross"], LAYER)["kx"]
    print(f"memory without the positional embedding: the smallest c a row needs at kx {float(need.min()):.3g} vs c {TM_C['kx']:.3g}")
    assert (need > TM_C["kx"]).all(), need
