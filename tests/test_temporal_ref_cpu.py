"""CPU: the fp64 temporal-transformer reference and the acceptance rule of tests/test_gpu_zz_temporal_ref.py, at the 7B layer
shapes (dim 4096, 32 heads, ffn 11264, text_card 32000, depformer_in 8 x 1024) with two layers and a 64-slot ring.

``temporal_layer_ref64`` (tests/util.py) restates one layer in float64 with the bf16 model's cast points, teacher-forced on
the implementation's own taps: each linear is judged on the implementation's input.  Shown here:

* The rule accepts a correct bf16 temporal transformer: the bf16 oracle (oracle/lm.py forward_text, fp32 accumulation in
  torch's order), whose activations are recorded at the same taps, passes every checkpoint of two steps at B = 4 and B = 256,
  with rings holding random history at positions 50..69 (the new keys land before and after the wrap at 64).  TM_C is at
  least about twice what it needs (the test prints both; tests/util.py says which constants the GPU handle set higher).  The
  int8 oracle (QLinear) gives x_attn and x_out bit for bit.
* The rule rejects layers with a bug: each mutant below computes a subtly wrong layer (at layer 1, step 1 of B = 256), and the
  checkpoint named beside it must reject it in every row the bug touches.

Not claimed: ulp-level cast-point mutants (a missing bf16 round of q, of the gate, or of the attention output).  Such a bug
moves a value by at most half a bf16 ulp, which the rule's 2^-7 relative term admits by design.

The synthetic weights keep |x| of the residual stream about 1.4 times the rms of an update; the residual checkpoints take
their rms from the update, so a lost k-block of out_proj / linear_out is still rejected (see the mutants).
"""
import contextlib
import dataclasses

import pytest
import torch

from moshi_b200.config import LMConfig
from moshi_b200.synth import iter_synth_lm_tensors
from oracle import quant
from oracle import transformer as tr
from oracle.lm import LMOracle, LMSpec
from tests.util import (TM_C, temporal_embed_ref64, temporal_heads_ref64, temporal_layer_ref64, tm_c_needed,
                        tm_layer_checkpoints, tm_row_ratios)

CFG = LMConfig(num_layers=2, context=64)
STEPS = 2
LAYER, STEP = 1, 1          # where the mutants act
KEEP = ("emb.", "text_emb.", "text_linear.", "out_norm.", "transformer.", "depformer_in.")


@pytest.fixture(scope="module")
def sd():
    return {k: v for k, v in iter_synth_lm_tensors(CFG, seed=23) if k.startswith(KEEP)}


@contextlib.contextmanager
def _recording(sd: dict, L: int):
    """Records the inputs of every temporal linear and norm the oracle runs: log of ((name, layer), x, y)."""
    names = {id(sd[f"transformer.layers.{l}.{k}"]): (n, l) for l in range(L)
             for n, k in (("in", "self_attn.in_projs.0.weight"), ("out", "self_attn.out_projs.0.weight"),
                          ("lin_in", "gating.linear_in.weight"), ("lin_out", "gating.linear_out.weight"))}
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


def _oracle_run(sd: dict, cfg: LMConfig, B: int, seed: int) -> list[dict]:
    """STEPS oracle steps of the temporal transformer with history in the rings; per step the taps, rings and heads."""
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, quantize=cfg.quantize)
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
    out = []
    for _ in range(STEPS):
        tok = torch.randint(0, cfg.card, (B, cfg.n_q + 1), generator=g)
        tok[::3, 5] = -1                                           # the zero row of an ungenerated stream
        before = [(ls.k.clone(), ls.v.clone()) for ls in st.layers]
        with _recording(sd, cfg.num_layers) as log:
            tout, logits = orc.forward_text(tok[:, :, None])
        taps = {key: x for key, x, _ in log if key[0] == "norm"}
        lins = {key: (x, y) for key, x, y in log if key[0] != "norm"}
        L = cfg.num_layers
        layers = []
        for l in range(L):
            nxt = taps[("norm", f"transformer.layers.{l + 1}.norm1")] if l + 1 < L else taps[("norm", "out_norm")]
            layers.append(dict(x_in=taps[("norm", f"transformer.layers.{l}.norm1")], attn_out=lins[("out", l)][0],
                               out_upd=lins[("out", l)][1], x_attn=taps[("norm", f"transformer.layers.{l}.norm2")],
                               gated=lins[("lin_out", l)][0], x_out=nxt,
                               ring=(st.layers[l].k.clone(), st.layers[l].v.clone()), ring_before=before[l]))
        tout = tout[:, 0]
        din = torch.stack([tr.linear(tout, sd[f"depformer_in.{k}.weight"], cfg.quantize) for k in range(cfg.dep_q)], dim=1)
        out.append(dict(tokens=tok, pos=pos.clone(), layers=layers, tout=tout, text_logits=logits[:, 0, 0], dep_in=din))
        pos = pos + 1
    return out


def _checkpoints(sd: dict, cfg: LMConfig, step: dict, mutant: dict | None = None, layers=None):
    """(name, kind, got, want, rms source) of one oracle step against the references, in the order the step computes them."""
    B = step["tokens"].shape[0]
    ex = torch.ones(B, dtype=torch.bool)
    pos = step["pos"]
    ar = torch.arange(B)
    L = step["layers"]
    out = [("embed", "embed", L[0]["x_in"], temporal_embed_ref64(sd, cfg, step["tokens"]), None)]
    for l in range(len(L)) if layers is None else layers:
        t = L[l]
        kr, vr = t["ring"]
        cap = kr.shape[2]
        want = temporal_layer_ref64(sd, cfg, l, t["x_in"], t["attn_out"], t["x_attn"], t["gated"], t["ring"], pos, ex, mutant)
        got = dict(k=kr[ar, :, pos % cap], v=vr[ar, :, pos % cap], attn_out=t["attn_out"], x_attn=t["x_attn"],
                   gated=t["gated"], x_out=t["x_out"])
        out += [(f"layer {l} {kind}", kind, g, w, s) for kind, g, w, s in tm_layer_checkpoints(want, got, ex)]
    heads = temporal_heads_ref64(sd, cfg, L[-1]["x_out"], step["tout"], mutant)
    out += [(k, k, step[k] if k != "transformer_out" else step["tout"], heads[k], None)
            for k in ("transformer_out", "text_logits", "dep_in")]
    return out


@pytest.fixture(scope="module")
def runs(sd):
    return {B: _oracle_run(sd, CFG, B, seed=B) for B in (4, 256)}


def test_bf16_oracle_passes_every_checkpoint(sd, runs):
    need, bad = {}, []
    for B, steps in runs.items():
        nb = {}
        for s, step in enumerate(steps):
            for name, kind, g, w, sc in _checkpoints(sd, CFG, step):
                nb[kind] = max(nb.get(kind, 0.0), tm_c_needed(g, w, sc))
                r = tm_row_ratios(g, w, kind, sc)
                if (r > 1).any():
                    bad.append((B, s, name, float(r.max())))
        print(f"\nB = {B}: c the bf16 oracle needs: " + ", ".join(f"{k} {v:.2e}" for k, v in nb.items()))
        for k, v in nb.items():
            need[k] = max(need.get(k, 0.0), v)
    print("c used: " + ", ".join(f"{k} {TM_C[k]:.2e} ({TM_C[k] / max(need[k], 1e-30):.1f}x)" for k in need))
    assert not bad, bad


def test_int8_oracle_residuals_are_exact(sd):
    """QLinear's integer products are exact, so given the taps x_attn and x_out match bit for bit; the rest passes the rule."""
    cfg = dataclasses.replace(CFG, quantize=True)
    steps = _oracle_run(sd, cfg, 4, seed=9)
    for s, step in enumerate(steps):
        for name, kind, g, w, sc in _checkpoints(sd, cfg, step):
            if kind in ("x_attn", "x_out"):
                assert torch.equal(g, w.bfloat16()), (s, name)
            assert not (tm_row_ratios(g, w, kind, sc) > 1).any(), (s, name)
    quant.clear_cache()


# ---- mutants ---------------------------------------------------------------------------------------------------------------
def _kblock(name: str, layer, kb: int = 5):
    """One 64-wide k-block (columns kb*64 .. kb*64+63) of the weight of one linear zeroed."""
    def f(n, ll, fetch):
        w = fetch(n, ll)
        if (n, ll) == (name, layer):
            w = w.clone()
            w[:, kb * 64:(kb + 1) * 64] = 0
        return w
    return {"weight": f}


def _on_linear(name: str, layer, fn):
    def f(n, ll, x, w, y):
        return fn(x, w, y.clone()) if (n, ll) == (name, layer) else y
    return {"linear": f}


def _stale_tile(prev_y: torch.Tensor, col: int = 3):
    def fn(x, w, y):
        y[:, col * 128:(col + 1) * 128] = prev_y[:, col * 128:(col + 1) * 128].double()
        return y
    return fn


def _segment_twice(x, w, y, tile: int = 1, k0: int = 1024, k1: int = 1536):
    c = slice(tile * 128, (tile + 1) * 128)
    y[:, c] += x[:, k0:k1].double() @ w[c, k0:k1].double().T
    return y


def _row_block(x, w, y):
    y[128:256] = x[0:128].double() @ w.double().T
    return y


def _swap_gate(x, w, y):
    F_ = y.shape[1] // 2
    return torch.cat([y[:, F_:], y[:, :F_]], dim=1)


def _swap_norms(layer):
    def f(n, ll, fetch):
        if ll == layer and n in ("n1", "n2"):
            return fetch("n2" if n == "n1" else "n1", ll)
        return fetch(n, ll)
    return {"weight": f}


ALL = slice(None)
MUTANTS = {
    # name: (mutant, checkpoint that must reject it, rows it touches)
    "k-block missing: in_proj": (_kblock("in", LAYER), "k", ALL),
    "k-block missing: out_proj": (_kblock("out", LAYER), "x_attn", ALL),
    "k-block missing: linear_in": (_kblock("lin_in", LAYER), "gated", ALL),
    "k-block missing: linear_out": (_kblock("lin_out", LAYER), "x_out", ALL),
    "k-block missing: text head": (_kblock("head", None), "text_logits", ALL),
    "k-block missing: depformer_in": (_kblock("din", 2), "dep_in", ALL),
    "output tile at the previous step's value": (None, "x_attn", ALL),
    "stream-K k-segment added twice": (_on_linear("lin_out", LAYER, _segment_twice), "x_out", ALL),
    "rows 128..255 with rows 0..127's activations": (_on_linear("lin_in", LAYER, _row_block), "gated", slice(128, 256)),
    "gate and value swapped": (_on_linear("lin_in", LAYER, _swap_gate), "gated", ALL),
    "attention residual dropped": ({"residual": lambda l, w: (l, w) != (LAYER, "attn")}, "x_attn", ALL),
    "MLP residual dropped": ({"residual": lambda l, w: (l, w) != (LAYER, "ffn")}, "x_out", ALL),
    "norm1 and norm2 alphas swapped": (_swap_norms(LAYER), "k", ALL),
    "k rotated at pos - 1": ({"rope_shift": -1}, "k", ALL),
    "k written one slot off": (None, "k", ALL),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_rejected_at_its_checkpoint_in_every_row(sd, runs, name):
    mutant, kind, rows = MUTANTS[name]
    step = runs[256][STEP]
    t = step["layers"][LAYER]
    if name == "output tile at the previous step's value":
        mutant = _on_linear("out", LAYER, _stale_tile(runs[256][STEP - 1]["layers"][LAYER]["out_upd"]))
    key = kind if kind in ("text_logits", "dep_in") else f"layer {LAYER} {kind}"
    _, w, s = {n: (g, w, s) for n, _, g, w, s in _checkpoints(sd, CFG, step, layers=[LAYER])}[key]
    if name == "k written one slot off":
        # the new key went to slot pos + 1: slot pos still holds what the ring held before the step
        kb = t["ring_before"][0]
        got = kb[torch.arange(kb.shape[0]), :, step["pos"] % kb.shape[2]]
    else:           # the mutant reference stands in for the implementation
        got = {n: w for n, _, _, w, _ in _checkpoints(sd, CFG, step, mutant, layers=[LAYER])}[key].bfloat16()
    r = tm_row_ratios(got, w, kind, s)
    print(f"{name}: rejected at {key}, smallest row ratio {float(r[rows].min()):.3g} "
          f"(rows {rows.start or 0}..{(rows.stop or r.numel()) - 1}), need {tm_c_needed(got, w, s):.3g} vs c {TM_C[kind]:.3g}")
    assert (r[rows] > 1).all(), (name, r[rows])


def test_int8_row_quantised_with_its_neighbours_scale_is_rejected(sd):
    """One row of out_proj's int8 activations quantised with the next row's absmax: x_attn is no longer bit-exact there."""
    cfg = dataclasses.replace(CFG, num_layers=1, quantize=True)
    step = _oracle_run(sd, cfg, 4, seed=11)[0]
    t = step["layers"][0]
    row = 1

    def neighbour(x, w, y):
        qw, sw = quant.cached_quantize_weight(w)
        xb = x.float()
        amax = xb.abs().amax(-1)
        q = torch.round(xb[row] * (127.0 / amax[row + 1])).clamp(-127, 127)
        acc = q.double() @ qw.double().T
        y[row] = (acc.float() * (amax[row + 1] * sw) * torch.tensor(float(quant.INV_127_SQ))).double()
        return y

    ex = torch.ones(4, dtype=torch.bool)
    want = temporal_layer_ref64(sd, cfg, 0, t["x_in"], t["attn_out"], t["x_attn"], t["gated"], t["ring"], step["pos"], ex)
    bad = temporal_layer_ref64(sd, cfg, 0, t["x_in"], t["attn_out"], t["x_attn"], t["gated"], t["ring"], step["pos"], ex,
                               _on_linear("out", 0, neighbour))
    differs = (bad["x_attn"].bfloat16() != want["x_attn"].bfloat16()).any(-1)
    print(f"int8 neighbour scale: x_attn rows differing {differs.tolist()}")
    assert differs.tolist() == [r == row for r in range(4)]
    quant.clear_cache()
