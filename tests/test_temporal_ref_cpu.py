"""CPU: the fp64 temporal-transformer reference and the acceptance rule of tests/test_gpu_zz_temporal_ref.py, at the 7B layer
shapes (dim 4096, 32 heads, ffn 11264, text_card 32000, depformer_in 8 x 1024) and at the 2B ones (tests/golden/
moshi_dev_2b.json: dim 2560, 20 heads, ffn 7040, RoPE period 1e5, 33 embedding tables plus a random condition_sum,
text_card 48000, depformer_in 16 x 1024), each with two layers and a 64-slot ring.

``temporal_layer_ref64`` (tests/util.py) restates one layer in float64 with the bf16 model's cast points, teacher-forced on
the implementation's own taps: each linear is judged on the implementation's input.  Shown here:

* The rule accepts a correct bf16 temporal transformer: the bf16 oracle (oracle/lm.py forward_text, fp32 accumulation in
  torch's order), whose activations are recorded at the same taps, passes every checkpoint of two steps at B = 4 and B = 256,
  with rings holding random history at positions 50..69 (the new keys land before and after the wrap at 64).  TM_C is at
  least about twice what it needs (the test prints both; tests/util.py says which constants the GPU handle set higher).  The
  int8 oracle (QLinear) gives x_attn and x_out bit for bit.
* The rule rejects layers with a bug: each mutant below computes a subtly wrong layer (at layer 1, step 1 of B = 256), and the
  checkpoint named beside it must reject it in every row the bug touches.  At the 2B shapes every mutant is rejected too, and
  so are the last k-block of out_proj (K 2560), of linear_out (K 7040), of depformer_in and of the text head, and gate tile
  54 of ffn 7040 paired with value tile 53.
* The summed embeddings are a chain of bf16 adds in the reference's order; the oracle matches temporal_embed_bf16 bit for
  bit at 17 and 33 tables, so the GPU test holds the device to it exactly as well as to the rule.
* The extra heads of the STT models (extra_heads_ref64, extra_heads_ratios): the bf16 oracle's step_with_extra_heads passes
  at B = 256 (dim 2048, four heads of six; worst ratio 0.57), and the rule rejects a head reading another head's weight rows
  and a lane's k-stride dropped from the dot product in every (head, row), and a softmax over E + 1 entries in every pair
  where it moves a probability by more than twice the tolerance (89 % of them, and 97 % are rejected; in the rest the extra logit lies so far
  below the row's largest that its share is under the logits' rounding).

Not claimed: ulp-level cast-point mutants (a missing bf16 round of q, of the gate, or of the attention output).  Such a bug
moves a value by at most half a bf16 ulp, which the rule's 2^-7 relative term admits by design.

The synthetic weights keep |x| of the residual stream about 1.4 times the rms of an update; the residual checkpoints take
their rms from the update, so a lost k-block of out_proj / linear_out is still rejected (see the mutants).
"""
import contextlib
import dataclasses
import json
import pathlib

import pytest
import torch

from moshi_b200.config import LMConfig
from moshi_b200.synth import iter_synth_lm_tensors
from oracle import quant
from oracle import transformer as tr
from oracle.lm import LMOracle, LMSpec
from tests.util import (TM_C, extra_heads_ratios, extra_heads_ref64, temporal_embed_bf16, temporal_embed_ref64, temporal_heads_ref64, temporal_layer_ref64,
                        tm_c_needed, tm_layer_checkpoints, tm_row_ratios)

CFG = LMConfig(num_layers=2, context=64)
# the 2B model (tests/golden/moshi_dev_2b.json: dim 2560, 20 heads, ffn 7040, text_card 48000, 32 + 1 embedding tables, RoPE
# period 1e5, depformer_in 16 x 1024) with two layers; its LUT conditioner is replaced by a random condition_sum
_2B = json.loads((pathlib.Path(__file__).parent / "golden" / "moshi_dev_2b.json").read_text())
CFG_2B = LMConfig.from_dict({**{k: v for k, v in _2B.items() if k not in ("conditioners", "fuser")}, "num_layers": 2,
                             "context": 64})
STEPS = 2
LAYER, STEP = 1, 1          # where the mutants act
KEEP = ("emb.", "text_emb.", "text_linear.", "out_norm.", "transformer.", "depformer_in.")


@pytest.fixture(scope="module")
def sd():
    return {k: v for k, v in iter_synth_lm_tensors(CFG, seed=23) if k.startswith(KEEP)}


@pytest.fixture(scope="module")
def sd_2b():
    return {k: v for k, v in iter_synth_lm_tensors(CFG_2B, seed=29) if k.startswith(KEEP)}


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


def _oracle_run(sd: dict, cfg: LMConfig, B: int, seed: int, cond: bool = False) -> list[dict]:
    """STEPS oracle steps of the temporal transformer with history in the rings; per step the taps, rings and heads.  ``cond``:
    a random condition_sum [B, dim] is added to the embeddings (lm.py:398-399)."""
    g = torch.Generator().manual_seed(seed)
    csum = (0.5 * torch.randn(B, cfg.dim, generator=g)).bfloat16() if cond else None
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, quantize=cfg.quantize,
                   condition_sum=None if csum is None else csum[:, None])
    orc.streaming(B)
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
        out.append(dict(tokens=tok, pos=pos.clone(), layers=layers, tout=tout, text_logits=logits[:, 0, 0], dep_in=din, cond=csum))
        pos = pos + 1
    return out


def _checkpoints(sd: dict, cfg: LMConfig, step: dict, mutant: dict | None = None, layers=None):
    """(name, kind, got, want, rms source) of one oracle step against the references, in the order the step computes them."""
    B = step["tokens"].shape[0]
    ex = torch.ones(B, dtype=torch.bool)
    pos = step["pos"]
    ar = torch.arange(B)
    L = step["layers"]
    out = [("embed", "embed", L[0]["x_in"], temporal_embed_ref64(sd, cfg, step["tokens"], step["cond"]), None)]
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


@pytest.fixture(scope="module")
def runs_2b(sd_2b):
    return {B: _oracle_run(sd_2b, CFG_2B, B, seed=B + 1, cond=True) for B in (4, 256)}


def _oracle_passes(sd: dict, cfg: LMConfig, runs: dict) -> None:
    need, bad = {}, []
    for B, steps in runs.items():
        nb = {}
        for s, step in enumerate(steps):
            for name, kind, g, w, sc in _checkpoints(sd, cfg, step):
                nb[kind] = max(nb.get(kind, 0.0), tm_c_needed(g, w, sc))
                r = tm_row_ratios(g, w, kind, sc)
                if (r > 1).any():
                    bad.append((B, s, name, float(r.max())))
        print(f"\nB = {B}: c the bf16 oracle needs: " + ", ".join(f"{k} {v:.2e}" for k, v in nb.items()))
        for k, v in nb.items():
            need[k] = max(need.get(k, 0.0), v)
    print("c used: " + ", ".join(f"{k} {TM_C[k]:.2e} ({TM_C[k] / max(need[k], 1e-30):.1f}x)" for k in need))
    assert not bad, bad


def test_bf16_oracle_passes_every_checkpoint(sd, runs):
    _oracle_passes(sd, CFG, runs)


def test_bf16_oracle_passes_every_checkpoint_at_2b(sd_2b, runs_2b):
    """The 2B shapes: in_proj N 7680, gate/value 2 x 7040 rows, linear_out K 7040, the text head N 48000, depformer_in 16 x
    1024, 20 heads at RoPE period 1e5, and 33 embeddings plus the condition sum in front of layer 0."""
    _oracle_passes(sd_2b, CFG_2B, runs_2b)


@pytest.mark.parametrize("geometry", ["7b", "2b"])
def test_embeddings_are_the_bf16_sum_in_the_reference_order(request, geometry):
    """The summed embeddings are a chain of bf16 adds in a fixed order (audio tables, text, condition sum), so an
    implementation that keeps that order matches temporal_embed_bf16 bit for bit: the oracle does, at 17 and at 33 tables."""
    sd, runs, cfg = ((request.getfixturevalue("sd"), request.getfixturevalue("runs"), CFG) if geometry == "7b" else
                     (request.getfixturevalue("sd_2b"), request.getfixturevalue("runs_2b"), CFG_2B))
    for B, steps in runs.items():
        for s, step in enumerate(steps):
            want = temporal_embed_bf16(sd, step["tokens"], step["cond"])
            assert torch.equal(step["layers"][0]["x_in"], want), (B, s)
    # the order matters: with the text table added first the sums differ, so the exact check tells the orders apart
    step = runs[256][0]
    tok = step["tokens"]
    first = temporal_embed_bf16(sd, torch.cat([tok[:, 1:], tok[:, :1]], dim=1), step["cond"])
    changed = int((first != step["layers"][0]["x_in"]).sum())
    print(f"{geometry}: elements that change when the text table is added first: {changed} of {first.numel()}")
    assert changed > 0


def _int8_exact(sd: dict, cfg: LMConfig) -> None:
    cfg = dataclasses.replace(cfg, quantize=True)
    steps = _oracle_run(sd, cfg, 4, seed=9)
    for s, step in enumerate(steps):
        for name, kind, g, w, sc in _checkpoints(sd, cfg, step):
            if kind in ("x_attn", "x_out"):
                assert torch.equal(g, w.bfloat16()), (s, name)
            assert not (tm_row_ratios(g, w, kind, sc) > 1).any(), (s, name)
    quant.clear_cache()


def test_int8_oracle_residuals_are_exact(sd):
    """QLinear's integer products are exact, so given the taps x_attn and x_out match bit for bit; the rest passes the rule."""
    _int8_exact(sd, CFG)


def test_int8_oracle_residuals_are_exact_at_2b(sd_2b):
    _int8_exact(sd_2b, CFG_2B)


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


def _pair_gate_tile(gate_tile: int, value_tile: int):
    """linear_in's gate tile ``gate_tile`` (128 rows) multiplied with value tile ``value_tile`` instead of its own."""
    def fn(x, w, y):
        F_ = y.shape[1] // 2
        y[:, F_ + gate_tile * 128:F_ + (gate_tile + 1) * 128] = y[:, F_ + value_tile * 128:F_ + (value_tile + 1) * 128].clone()
        return y
    return fn


# at the 2B shapes, also the last k-block of the K extents no other model has (the one a wrong K partition drops) and the
# last of the 55 gate/value tile pairs of ffn 7040 paired with its neighbour
MUTANTS_2B = {
    **MUTANTS,
    "last k-block missing: out_proj (K 2560)": (_kblock("out", LAYER, 2560 // 64 - 1), "x_attn", ALL),
    "last k-block missing: linear_out (K 7040)": (_kblock("lin_out", LAYER, 7040 // 64 - 1), "x_out", ALL),
    "last k-block missing: depformer_in (K 2560)": (_kblock("din", 15, 2560 // 64 - 1), "dep_in", ALL),
    "last k-block missing: text head (K 2560)": (_kblock("head", None, 2560 // 64 - 1), "text_logits", ALL),
    "gate tile 54 with value tile 53": (_on_linear("lin_in", LAYER, _pair_gate_tile(54, 53)), "gated", ALL),
}


def _mutant_rejected(sd: dict, cfg: LMConfig, runs: dict, name: str, mutants: dict) -> None:
    mutant, kind, rows = mutants[name]
    step = runs[256][STEP]
    t = step["layers"][LAYER]
    if name == "output tile at the previous step's value":
        mutant = _on_linear("out", LAYER, _stale_tile(runs[256][STEP - 1]["layers"][LAYER]["out_upd"]))
    key = kind if kind in ("text_logits", "dep_in") else f"layer {LAYER} {kind}"
    _, w, s = {n: (g, w, s) for n, _, g, w, s in _checkpoints(sd, cfg, step, layers=[LAYER])}[key]
    if name == "k written one slot off":
        # the new key went to slot pos + 1: slot pos still holds what the ring held before the step
        kb = t["ring_before"][0]
        got = kb[torch.arange(kb.shape[0]), :, step["pos"] % kb.shape[2]]
    else:           # the mutant reference stands in for the implementation
        got = {n: w for n, _, _, w, _ in _checkpoints(sd, cfg, step, mutant, layers=[LAYER])}[key].bfloat16()
    r = tm_row_ratios(got, w, kind, s)
    print(f"{name}: rejected at {key}, smallest row ratio {float(r[rows].min()):.3g} "
          f"(rows {rows.start or 0}..{(rows.stop or r.numel()) - 1}), need {tm_c_needed(got, w, s):.3g} vs c {TM_C[kind]:.3g}")
    assert (r[rows] > 1).all(), (name, r[rows])


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_rejected_at_its_checkpoint_in_every_row(sd, runs, name):
    _mutant_rejected(sd, CFG, runs, name, MUTANTS)


@pytest.mark.parametrize("name", list(MUTANTS_2B))
def test_mutant_rejected_at_2b_shapes(sd_2b, runs_2b, name):
    _mutant_rejected(sd_2b, CFG_2B, runs_2b, name, MUTANTS_2B)


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


# ---- the extra heads of the STT models -------------------------------------------------------------------------------------
# the STT geometry of tests/test_gpu_zz_temporal_ref.py ("stt": dim 2048, 16 heads, n_q 32, dep_q 0, text_card 8000, four
# extra heads of six outputs) with one layer
CFG_STT = LMConfig(dim=2048, num_heads=16, num_layers=1, context=64, n_q=32, dep_q=0, text_card=8000, delays=[0] * 33,
                   extra_heads_num_heads=4, extra_heads_dim=6)


@pytest.fixture(scope="module")
def stt_step():
    """The second step of the bf16 oracle's step_with_extra_heads at B = 256: (sd, its transformer_out [B, dim], its heads [n, B, E])."""
    sd = dict(iter_synth_lm_tensors(CFG_STT, seed=37))
    spec = dataclasses.replace(LMSpec.from_config(CFG_STT), extra_heads_num_heads=CFG_STT.extra_heads_num_heads,
                               extra_heads_dim=CFG_STT.extra_heads_dim)
    orc = LMOracle(sd, spec, use_sampling=False)
    B = 256
    orc.streaming(B)
    g = torch.Generator().manual_seed(3)
    for _ in range(2):                      # the first step feeds every row the initial tokens
        _, heads = orc.step_with_extra_heads(torch.randint(0, CFG_STT.card, (B, CFG_STT.n_q, 1), generator=g))
    return sd, orc.last_transformer_out[:, 0], torch.stack([h[:, 0] for h in heads])


def test_bf16_oracle_extra_heads_pass_the_rule(stt_step):
    sd, tout, got = stt_step
    ref = extra_heads_ref64(sd, CFG_STT, tout)
    assert torch.equal(temporal_heads_ref64(sd, CFG_STT, tout, tout)["extra_heads"]["p"], ref["p"])
    r = extra_heads_ratios(got, ref)
    print(f"\nextra heads of the bf16 oracle at B = {tout.shape[0]}: worst ratio {float(r.max()):.3f}, "
          f"(head, row) pairs off the reference's bf16 probability {int((got != ref['p'].bfloat16()).any(-1).sum())} "
          f"of {r.numel()}")
    assert not (r > 1).any(), r.max()


def _other_head(i, fetch):
    return fetch((i + 1) % CFG_STT.extra_heads_num_heads)


def _lane_dropped(i, fetch, lane: int = 31):
    w = fetch(i).clone()
    w[:, lane::32] = 0                      # the terms one lane of the warp sums: k = lane, lane + 32, ...
    return w


def _one_more_entry(lg):
    # lane E's logit would be row 0 of the next head's weight, which follows the head's E rows in memory
    return torch.cat([lg, lg.roll(-1, dims=0)[..., :1]], dim=-1)


EXTRA_MUTANTS = {
    "head reading another head's weight rows": {"weight": _other_head},
    "lane 31's k-stride dropped from the dot product": {"weight": _lane_dropped},
    # the extra entry moves every probability by the share p_extra it takes; where its logit lies far below the row's
    # largest that share is below the rounding of the logits, and the rule cannot see it there
    "softmax over E + 1 entries": {"logits": _one_more_entry},
}


@pytest.mark.parametrize("name", list(EXTRA_MUTANTS))
def test_extra_heads_mutant_rejected(stt_step, name):
    """Rejected in every (head, row) where the mutant moves a probability by more than twice the tolerance before its bf16
    rounding (which moves it by at most the tolerance's half-ulp term): every pair for the first two mutants."""
    sd, tout, _ = stt_step
    ref = extra_heads_ref64(sd, CFG_STT, tout)
    bad = extra_heads_ref64(sd, CFG_STT, tout, EXTRA_MUTANTS[name])["p"]
    r = extra_heads_ratios(bad.bfloat16(), ref)
    visible = extra_heads_ratios(bad, ref) > 2
    print(f"{name}: rejected in {float((r > 1).double().mean()):.1%} of the (head, row) pairs, moved by more than twice the "
          f"tolerance in {float(visible.double().mean()):.1%}, smallest ratio {float(r.min()):.3g}")
    assert (r[visible] > 1).all(), name
    if name != "softmax over E + 1 entries":
        assert visible.all(), name
    else:
        assert float(visible.double().mean()) > 0.85, name        # 89 % of the pairs at these weights
