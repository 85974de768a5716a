"""CPU: the fp64 depformer reference and the acceptance rule of tests/test_gpu_zz_depformer_ref.py, at the 7B depformer shapes
and at the 2B model's depformer (the same layer shapes over dep_q 16 sub-steps, depformer_in with K 2560).

``depformer_ref64`` restates one frame of the depformer in float64 with the bf16 model's cast points.  Two things are shown here:

* The rule accepts a correct bf16 depformer: the bf16 oracle (oracle/lm.py, fp32 accumulation in torch's order) passes at every
  checkpoint of two frames.  The constants of the rule (tests/util.py DEP_C_*) are about twice what the oracle needs.
* The rule rejects depformers with a bug that leaves the greedy tokens mostly intact: each mutant below computes a subtly wrong
  frame, and the checkpoint named beside it must reject it in every batch row.  The mutants sit at sub-step 3 and layer 2 of 6
  unless said otherwise, so that keys before and after the newest one exist and the error has layers to cross.

At the 2B depformer the oracle passes every layer at all 16 sub-steps (and layer 0 at B = 256), and a newest or first key
dropped from sub-step 14's attention (15 keys), the last k-block of depformer_in, sub-step 13's weights or embedding table
in sub-step 14 and a lost k-block of sub-step 15's head are each rejected in every row.

Not claimed: ulp-level cast-point mutants (a missing bf16 round of the gate, of q, or of the attention output).  Such a bug moves
a value by at most half a bf16 ulp, which is what the rule's 2^-7 relative term admits by design.

Where a mutant is caught, and by how much (the smallest c over the rows that would still admit it, against the constant):
the newest key or key 0 dropped 0.42 / 0.05 at the next layer's k; one k-block of in_proj 0.75 / 0.04 at the layer's own k, of
out_proj 0.19 / 0.05, of the gate/value input 0.26 / 0.05 and of linear_out 0.12 / 0.05 at the next layer's k, of the head
0.77 / 0.08 at the logits; another sub-step's weights 4.4 / 0.04; the previous sub-step's embedding table 0.13 / 0.004 and the
previous-but-one token 0.13 / 0.004 at layer 0; norm2's alpha in norm1 0.25 / 0.04, norm1's in norm2 0.069 / 0.05; a residual
not added 3.5 / 0.05.  A k-block missing from the LAST layer's linear_out only reaches the logits, where it moves them by 0.05
to 0.1 rms, about the logits constant: it is not rejected in every row, so the mutant sits at layer 2, where the next layer's k
rejects it.

int8 (quantize=True): the int8 oracle (oracle/quant.py's QLinear in every linear) passes depformer_ref64(quantize=True) at every
checkpoint, din bit for bit, under the DEP_C_*_I8 constants, on weights whose rows carry unequal int8 scales (dep_row_scaled:
synthetic uniform weights give every row, linear and sub-step the same scale, which would hide a scale read from the wrong
one).  Its mutants sit in layer 0, whose k / v the int8 oracle matches within the relative term: an activation row paired with
its neighbour row's scale, another sub-step's weight scales, a truncating quantiser and a lost 128-wide int8 k-block of in_proj
are rejected at layer 0's k (smallest admitting c 0.09 to 2.6, against 2^-7); a lost k-block of gate/value in or of linear_out
at layer 1's k (0.79 and 0.27, against 0.25) and of the head at the logits (1.6 against 0.5).  Not claimed: the gate and value
scales swapped, which needs only 0.245 at layer 1's k, below the 0.25 set there (twice the 0.126 the int8 oracle needs).

Classifier-free guidance: the bf16 oracle's depformer_step with cfg_coef = 3 over 2B rows passes at every checkpoint of both
halves with the bf16 constants, and its guided logits equal cfg_guide_bf16 of its model logits bit for bit.  Rejected in every
row: the null rows fed the conditioned rows' transformer_out (at din), the null rows given another row's previous token (at
layer 0's k), and, at the bit-exact guided logits, the combination with the halves swapped or with the previous sub-step's null
logits.
"""
import dataclasses
import json
import pathlib

import pytest
import torch

from moshi_b200.config import LMConfig
from moshi_b200.synth import iter_synth_lm_tensors
from oracle import transformer as tr
from oracle.lm import LMOracle, LMSpec, scaled_embedding
from tests.util import (DEP_C_DIN, DEP_C_LOGITS, DEP_C_LOGITS_I8, c_needed, cfg_guide64, cfg_guide_bf16, dep_c, dep_c_kv,
                        dep_checkpoints,
                        dep_row_ratios, dep_row_scaled, depformer_ref64, exact_row_ratios, greedy_unexcused)

# the 7B depformer (dd 1024, 16 heads, ffn 2816, 6 layers, dep_q 8, card 2048) behind a 4096-wide temporal output
CFG = LMConfig(num_layers=1, context=16)
# the 2B model's depformer (tests/golden/moshi_dev_2b.json: the same layer shapes, but dep_q 16 sub-steps with
# depformer_context 16, so the last sub-steps attend over up to 16 keys, and depformer_in reads a 2560-wide transformer_out)
_2B = json.loads((pathlib.Path(__file__).parent / "golden" / "moshi_dev_2b.json").read_text())
CFG_2B = LMConfig.from_dict({**{k: v for k, v in _2B.items() if k not in ("conditioners", "fuser")}, "num_layers": 1,
                             "context": 16})
B, FRAMES = 4, 2
K, LAYER = 3, 2          # where the mutants act
K_2B = 14                # where the 2B mutants act: 15 keys in the sub-step's attention


def _dep_sd(cfg: LMConfig, seed: int) -> dict:
    return {k: v for k, v in iter_synth_lm_tensors(cfg, seed=seed) if k.startswith(("depformer", "linears."))}


@pytest.fixture(scope="module")
def sd():
    return _dep_sd(CFG, 21)


@pytest.fixture(scope="module")
def sd_2b():
    return _dep_sd(CFG_2B, 22)


def _oracle_frame(orc: LMOracle, sd: dict, tout: torch.Tensor, text_token: torch.Tensor) -> tuple[dict, torch.Tensor]:
    """One frame of the oracle (bf16, or int8 with orc.quantize), greedy, with its per-frame cache kept: (checkpoints in
    depformer_ref64's layout, the audio tokens [dep_q, B] it sampled)."""
    st = tr.init_state(orc.dep_spec, tout.shape[0], torch.bfloat16)
    prev, toks, logits = text_token, [], []
    for k in range(orc.spec.dep_q):
        lg = orc.forward_depformer(k, prev[:, None], tout[:, None], st)[:, 0, 0]
        logits.append(lg)
        prev = lg.float().argmax(-1)
        toks.append(prev)
    din = torch.stack([tr.linear(tout, sd[f"depformer_in.{k}.weight"], orc.quantize) for k in range(orc.spec.dep_q)], dim=1)
    got = dict(din=din, k=[ls.k for ls in st.layers], v=[ls.v for ls in st.layers], logits=torch.stack(logits))
    return got, torch.stack(toks)


def _frames(sd: dict, cfg: LMConfig, seed: int) -> list:
    orc = LMOracle({**sd, "text_emb.weight": torch.zeros(1, dtype=torch.bfloat16)}, LMSpec.from_config(cfg), use_sampling=False)
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(FRAMES):
        tout = torch.randn(B, cfg.dim, generator=g).bfloat16()
        text = torch.randint(0, cfg.text_card, (B,), generator=g)
        got, toks = _oracle_frame(orc, sd, tout, text)
        out.append((tout, text, toks, got, depformer_ref64(sd, cfg, tout, text, toks)))
    return out


@pytest.fixture(scope="module")
def frames(sd):
    """Per frame: (transformer_out, text token, the oracle's tokens, the oracle's checkpoints, depformer_ref64 of the frame)."""
    return _frames(sd, CFG, 5)


@pytest.fixture(scope="module")
def frames_2b(sd_2b):
    return _frames(sd_2b, CFG_2B, 4)


def _oracle_passes(frames_: list) -> None:
    need = {}
    for _, _, _, got, want in frames_:
        for kind, k, layer, g, w in dep_checkpoints(got, want):
            key = kind if kind in ("din", "logits") else f"kv{layer}"
            need[key] = max(need.get(key, 0.0), c_needed(g, w))
            bad = dep_row_ratios(g, w, kind, layer) > 1
            assert not bad.any(), (kind, k, layer, dep_row_ratios(g, w, kind, layer))
    print("c the bf16 oracle needs: " + ", ".join(f"{k} {v:.4f}" for k, v in need.items()))
    print(f"c used: din {DEP_C_DIN}, kv {[dep_c_kv(l) for l in range(CFG.depformer_num_layers)]}, logits {DEP_C_LOGITS}")


def test_bf16_oracle_passes_every_checkpoint(frames):
    _oracle_passes(frames)


def test_bf16_oracle_passes_every_checkpoint_at_2b(frames_2b):
    """All six layers at all 16 sub-steps of the 2B depformer."""
    _oracle_passes(frames_2b)


def _layer0_at_serving_batch(sd: dict, cfg: LMConfig, seed: int) -> None:
    Bs = 256
    g = torch.Generator().manual_seed(seed)
    need = 0.0
    for _ in range(FRAMES):
        tout = torch.randn(Bs, cfg.dim, generator=g).bfloat16()
        text = torch.randint(0, cfg.text_card, (Bs,), generator=g)
        toks = torch.randint(0, cfg.card, (cfg.dep_q, Bs), generator=g)
        want = depformer_ref64(sd, dataclasses.replace(cfg, depformer_num_layers=1), tout, text, toks)
        prev = [text] + list(toks[:-1])
        for k in range(cfg.dep_q):
            emb = scaled_embedding(sd, "depformer_text_emb" if k == 0 else f"depformer_emb.{k - 1}", prev[k])
            x = tr.linear(tout, sd[f"depformer_in.{k}.weight"]) + emb
            xn = tr.apply_norm("rms_norm_f32", x[:, None], sd, "depformer.layers.0.norm1")[:, 0]
            qkv = tr.linear(xn, sd[f"depformer.layers.0.self_attn.in_projs.{k}.weight"]).view(Bs, 3, cfg.depformer_num_heads, 64)
            for i, kind in ((1, "k"), (2, "v")):
                w = want[kind][0][:, :, k]
                need = max(need, c_needed(qkv[:, i], w))
                assert not (dep_row_ratios(qkv[:, i], w, kind, 0) > 1).any(), (kind, k)
    print(f"layer 0 at B = {Bs}: c the bf16 oracle needs {need:.4f}, c used {dep_c_kv(0)}")


def test_bf16_oracle_passes_layer0_at_serving_batch(sd):
    """Layer 0's k / v at B = 256: only din, the embedding, RMSNorm and in_proj precede them, so their rare rounding flips are
    sampled here over as many rows as the fused kernel serves (the oracle's own ops, against depformer_ref64 restricted to
    layer 0, random tokens)."""
    _layer0_at_serving_batch(sd, CFG, 7)


def test_bf16_oracle_passes_layer0_at_serving_batch_at_2b(sd_2b):
    """As above for the 2B depformer: 16 sub-steps, depformer_in with K 2560."""
    _layer0_at_serving_batch(sd_2b, CFG_2B, 8)


def _kblock(name: str, k: int, layer, kb: int = 5):
    """The weight of one GEMM with one 64-wide k-block (columns kb*64 .. kb*64+63) zeroed."""
    def f(n, kk, ll, fetch):
        w = fetch(n, kk, ll)
        if (n, kk, ll) == (name, k, layer):
            w = w.clone()
            w[:, kb * 64:(kb + 1) * 64] = 0
        return w
    return {"weight": f}


def _swap(sub: dict):
    """Replace the fetch of (name, k, layer) by another: sub maps (name, k, layer or None) -> (name, k, layer)."""
    def f(n, kk, ll, fetch):
        return fetch(*sub.get((n, kk, ll), (n, kk, ll)))
    return {"weight": f}


L = CFG.depformer_num_layers
MUTANTS = {
    # name: (mutant, (checkpoint kind, sub-step, layer) that must reject it in every row)
    "newest key dropped": ({"keys": lambda k, l: (0, k) if (k, l) == (K, LAYER) else (0, k + 1)}, ("k", K, LAYER + 1)),
    "key 0 dropped": ({"keys": lambda k, l: (1, k + 1) if (k, l) == (K, LAYER) else (0, k + 1)}, ("k", K, LAYER + 1)),
    "k-block missing: in_proj": (_kblock("in", K, LAYER), ("k", K, LAYER)),
    "k-block missing: out_proj": (_kblock("out", K, LAYER), ("k", K, LAYER + 1)),
    "k-block missing: gate/value in": (_kblock("lin_in", K, LAYER), ("k", K, LAYER + 1)),
    "k-block missing: linear_out": (_kblock("lin_out", K, LAYER), ("k", K, LAYER + 1)),
    "k-block missing: head": (_kblock("head", K, None), ("logits", K, None)),
    "sub-step k-1 weights in one layer": (_swap({(n, K, LAYER): (n, K - 1, LAYER) for n in ("in", "out", "lin_in", "lin_out")}),
                                          ("k", K, LAYER)),
    "embedding table of sub-step k-1": (_swap({("emb", K, None): ("emb", K - 1, None)}), ("k", K, 0)),
    "previous-but-one token": ({"prev": lambda k, t: t[k - 1] if k == K else t[k]}, ("k", K, 0)),
    "norm2 alpha in norm1": (_swap({("n1", k, LAYER): ("n2", k, LAYER) for k in range(CFG.dep_q)}), ("k", 0, LAYER)),
    "norm1 alpha in norm2": (_swap({("n2", k, LAYER): ("n1", k, LAYER) for k in range(CFG.dep_q)}), ("k", 0, LAYER + 1)),
    "attention residual not added": ({"residual": lambda k, l, w: (k, l, w) != (K, LAYER, "attn")}, ("k", K, LAYER + 1)),
    "ffn residual not added": ({"residual": lambda k, l, w: (k, l, w) != (K, LAYER, "ffn")}, ("k", K, LAYER + 1)),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_rejected_at_its_checkpoint_in_every_row(sd, frames, name):
    mutant, (kind, k, layer) = MUTANTS[name]
    tout, text, toks, _, want = frames[0]
    if name == "previous-but-one token":
        assert (toks[K - 1] != toks[K - 2]).all()            # else the mutant computes the right frame for that row
    bad = depformer_ref64(sd, CFG, tout, text, toks, mutant)
    got = {n: [t.bfloat16() for t in v] if isinstance(v, list) else v.bfloat16() for n, v in bad.items()}
    cps = {(kd, kk, ll): (g, w) for kd, kk, ll, g, w in dep_checkpoints(got, want)}
    r = dep_row_ratios(*cps[(kind, k, layer)], kind, layer)
    print(f"{name}: rejected at {kind} sub-step {k} layer {layer}, row ratios {[round(float(x), 2) for x in r]}")
    assert (r > 1).all(), (name, r)


MUTANTS_2B = {
    # at sub-step 14 of 16, where 15 keys are in the attention
    "newest key dropped": ({"keys": lambda k, l: (0, k) if (k, l) == (K_2B, LAYER) else (0, k + 1)}, ("k", K_2B, LAYER + 1)),
    "key 0 dropped": ({"keys": lambda k, l: (1, k + 1) if (k, l) == (K_2B, LAYER) else (0, k + 1)}, ("k", K_2B, LAYER + 1)),
    "last k-block missing: depformer_in (K 2560)": (_kblock("din", 15, None, 2560 // 64 - 1), ("din", 15, None)),
    "sub-step k-1 weights in one layer": (_swap({(n, K_2B, LAYER): (n, K_2B - 1, LAYER)
                                                 for n in ("in", "out", "lin_in", "lin_out")}), ("k", K_2B, LAYER)),
    "embedding table of sub-step k-1": (_swap({("emb", K_2B, None): ("emb", K_2B - 1, None)}), ("k", K_2B, 0)),
    "k-block missing: head of sub-step 15": (_kblock("head", 15, None), ("logits", 15, None)),
}


@pytest.mark.parametrize("name", list(MUTANTS_2B))
def test_mutant_rejected_at_2b_shapes(sd_2b, frames_2b, name):
    mutant, (kind, k, layer) = MUTANTS_2B[name]
    tout, text, toks, _, want = frames_2b[0]
    bad = depformer_ref64(sd_2b, CFG_2B, tout, text, toks, mutant)
    got = {n: [t.bfloat16() for t in v] if isinstance(v, list) else v.bfloat16() for n, v in bad.items()}
    cps = {(kd, kk, ll): (g, w) for kd, kk, ll, g, w in dep_checkpoints(got, want)}
    r = dep_row_ratios(*cps[(kind, k, layer)], kind, layer)
    print(f"2B {name}: rejected at {kind} sub-step {k} layer {layer}, row ratios {[round(float(x), 2) for x in r]}")
    assert (r > 1).all(), (name, r)


# ---- int8: LMModel(quantize=True), every depformer linear a QLinear --------------------------------------------------------
def _kinds_needed(frames_: list, need: dict) -> None:
    for _, _, _, got, want in frames_:
        for kind, k, layer, g, w in dep_checkpoints(got, want):
            key = kind if kind in ("din", "logits") else f"kv{layer}"
            need[key] = max(need.get(key, 0.0), c_needed(g, w))


@pytest.fixture(scope="module")
def qsd(sd):
    return dep_row_scaled(sd, seed=3)


@pytest.fixture(scope="module")
def qframes(qsd):
    """As ``frames``, for the int8 oracle (oracle/quant.py's QLinear in every linear) against depformer_ref64(quantize=True), on
    weights whose rows have unequal int8 scales (dep_row_scaled)."""
    sd = qsd
    orc = LMOracle({**sd, "text_emb.weight": torch.zeros(1, dtype=torch.bfloat16)}, LMSpec.from_config(CFG), use_sampling=False,
                   quantize=True)
    g = torch.Generator().manual_seed(6)
    out = []
    for _ in range(FRAMES):
        tout = torch.randn(B, CFG.dim, generator=g).bfloat16()
        text = torch.randint(0, CFG.text_card, (B,), generator=g)
        got, toks = _oracle_frame(orc, sd, tout, text)
        out.append((tout, text, toks, got, depformer_ref64(sd, CFG, tout, text, toks, quantize=True)))
    return out


def test_int8_oracle_passes_every_checkpoint(qframes):
    """din is exact given transformer_out (one QLinear of a bf16 input), so it must match bit for bit; every other checkpoint
    is held to the bf16 rule."""
    need = {}
    for _, _, _, got, want in qframes:
        for kind, k, layer, g, w in dep_checkpoints(got, want):
            r = exact_row_ratios(g, w) if kind == "din" else dep_row_ratios(g, w, kind, layer, int8=True)
            assert not (r > 1).any(), (kind, k, layer, r)
    _kinds_needed(qframes, need)
    print("c the int8 oracle needs: " + ", ".join(f"{k} {v:.4f}" for k, v in need.items()))
    print(f"c used: din exact, kv {[dep_c_kv(l, True) for l in range(CFG.depformer_num_layers)]}, logits {DEP_C_LOGITS_I8}")


def _int8_layer0_at_serving_batch(sd: dict, cfg: LMConfig, seed: int) -> None:
    from oracle.quant import qlinear
    Bs = 256
    g = torch.Generator().manual_seed(seed)
    need = 0.0
    for _ in range(FRAMES):
        tout = torch.randn(Bs, cfg.dim, generator=g).bfloat16()
        text = torch.randint(0, cfg.text_card, (Bs,), generator=g)
        toks = torch.randint(0, cfg.card, (cfg.dep_q, Bs), generator=g)
        want = depformer_ref64(sd, dataclasses.replace(cfg, depformer_num_layers=1), tout, text, toks, quantize=True)
        prev = [text] + list(toks[:-1])
        for k in range(cfg.dep_q):
            emb = scaled_embedding(sd, "depformer_text_emb" if k == 0 else f"depformer_emb.{k - 1}", prev[k])
            din = qlinear(tout, sd[f"depformer_in.{k}.weight"])
            assert torch.equal(din, want["din"][:, k].bfloat16()), k
            x = din + emb
            xn = tr.apply_norm("rms_norm_f32", x[:, None], sd, "depformer.layers.0.norm1")[:, 0]
            qkv = qlinear(xn, sd[f"depformer.layers.0.self_attn.in_projs.{k}.weight"]).view(Bs, 3, cfg.depformer_num_heads, 64)
            for i, kind in ((1, "k"), (2, "v")):
                w = want[kind][0][:, :, k]
                need = max(need, c_needed(qkv[:, i], w))
                assert not (dep_row_ratios(qkv[:, i], w, kind, 0, int8=True) > 1).any(), (kind, k)
    print(f"int8 layer 0 at B = {Bs}: c the int8 oracle needs {need:.4f}, c used {dep_c_kv(0, True)}")


def test_int8_oracle_passes_layer0_at_serving_batch(qsd):
    """Layer 0's k / v of the int8 oracle at B = 256, as test_bf16_oracle_passes_layer0_at_serving_batch does for bf16."""
    _int8_layer0_at_serving_batch(qsd, CFG, 8)


def test_int8_oracle_passes_layer0_at_serving_batch_at_2b(sd_2b):
    """The same at the 2B depformer: 16 sub-steps, depformer_in with K 2560."""
    _int8_layer0_at_serving_batch(dep_row_scaled(sd_2b, seed=3), CFG_2B, 9)


def _qat(name: str, k: int, layer, f):
    """A "qlinear" mutant that changes the quantised operands of one linear: f(x, q) -> q."""
    def g(n, kk, ll, x, q):
        return f(x, q) if (n, kk, ll) == (name, k, layer) else q
    return {"qlinear": g}


def _neighbour_scale(x, q):
    return {**q, "sa": q["sa"].roll(-1)}                     # row b's integers dequantised with row b + 1's scale


def _qkblock(x, q, kb: int = 5):
    qx = q["qx"].clone()
    qx[:, kb * 128:(kb + 1) * 128] = 0                          # one 128-byte int8 k-block of every row lost
    return {**q, "qx": qx}


def _gate_value_swapped(x, q):
    F_ = q["sw"].numel() // 2
    return {**q, "sw": torch.cat([q["sw"][F_:], q["sw"][:F_]])}


def _truncating(x, q):
    t = x.float()
    absmax = t.abs().amax(dim=-1)
    inv = torch.where(absmax > 0, torch.tensor(127.0, dtype=torch.float32) / absmax, torch.zeros_like(absmax))
    return {**q, "qx": torch.trunc(t * inv[:, None]).clamp_(-127, 127).to(torch.int8)}


def _other_step_scales(sd, name: str, layer):
    from oracle.quant import cached_quantize_weight
    from tests.util import _dep_tensor
    return lambda x, q: {**q, "sw": cached_quantize_weight(_dep_tensor(sd, name, K - 1, layer))[1]}


QMUTANTS = {
    # name: (mutant of sd, (checkpoint kind, sub-step, layer) that must reject it in every row).  The int8 mutants sit in layer
    # 0, whose k / v the int8 oracle matches to the relative term (c 2^-8), or act on its output at layer 1.
    "activation row with its neighbour row's scale: in_proj": (lambda sd: _qat("in", K, 0, _neighbour_scale), ("k", K, 0)),
    "weight scales of sub-step k-1: in_proj": (lambda sd: _qat("in", K, 0, _other_step_scales(sd, "in", 0)), ("k", K, 0)),
    "int8 k-block missing: in_proj": (lambda sd: _qat("in", K, 0, _qkblock), ("k", K, 0)),
    "int8 k-block missing: gate/value in": (lambda sd: _qat("lin_in", K, 0, _qkblock), ("k", K, 1)),
    "int8 k-block missing: linear_out": (lambda sd: _qat("lin_out", K, 0, _qkblock), ("k", K, 1)),
    "int8 k-block missing: head": (lambda sd: _qat("head", K, None, _qkblock), ("logits", K, None)),
    "quantiser truncating: in_proj": (lambda sd: _qat("in", K, 0, _truncating), ("k", K, 0)),
}


# Not claimed: measured where they would be caught, but admitted by the constant set there.
QMUTANTS_NOT_CLAIMED = {
    "gate and value scales swapped": (lambda sd: _qat("lin_in", K, 0, _gate_value_swapped), ("k", K, 1)),
}


@pytest.mark.parametrize("name", list(QMUTANTS) + list(QMUTANTS_NOT_CLAIMED))
def test_int8_mutant_rejected_at_its_checkpoint_in_every_row(qsd, qframes, name):
    sd = qsd
    make, (kind, k, layer) = {**QMUTANTS, **QMUTANTS_NOT_CLAIMED}[name]
    tout, text, toks, _, want = qframes[0]
    bad = depformer_ref64(sd, CFG, tout, text, toks, make(sd), quantize=True)
    got = {n: [t.bfloat16() for t in v] if isinstance(v, list) else v.bfloat16() for n, v in bad.items()}
    cps = {(kd, kk, ll): (g, w) for kd, kk, ll, g, w in dep_checkpoints(got, want)}
    g, w = cps[(kind, k, layer)]
    r = dep_row_ratios(g, w, kind, layer, int8=True)
    need = min(c_needed(g[b:b + 1], w[b:b + 1]) for b in range(B))
    print(f"{name}: rejected at {kind} sub-step {k} layer {layer}, row ratios {[round(float(x), 2) for x in r]}, "
          f"smallest c admitting it {need:.3f} / {dep_c(kind, layer, True)}"
          f"{' (not claimed)' if name in QMUTANTS_NOT_CLAIMED else ''}")
    if name not in QMUTANTS_NOT_CLAIMED:
        assert (r > 1).all(), (name, r)


# ---- classifier-free guidance: 2B model rows, the samplers read the guided B rows ------------------------------------------
COEF = 3.0


@pytest.fixture(scope="module")
def cfg_frames(sd):
    """Per frame of the bf16 oracle's depformer_step with cfg_coef = 3 over 2B rows: (transformer_out [2B, dim], text token
    [B], tokens [dep_q, B], checkpoints over 2B rows with the model's own logits, guided logits [dep_q, B, card] of the step,
    depformer_ref64 of the 2B rows teacher-forced on the tokens repeated for the null half, as lm.py:826-832 feeds them)."""
    orc = LMOracle({**sd, "text_emb.weight": torch.zeros(1, dtype=torch.bfloat16)}, LMSpec.from_config(CFG), use_sampling=False,
                   cfg_coef=COEF, cfg_is_no_text=True)
    g = torch.Generator().manual_seed(9)
    out = []
    for _ in range(FRAMES):
        tout = torch.randn(2 * B, CFG.dim, generator=g).bfloat16()
        text = torch.randint(0, CFG.text_card, (B,), generator=g)
        rec, guided = {"model": []}, []
        forward = orc.forward_depformer

        def recording(k, prev, transformer_out, st):
            lg = forward(k, prev, transformer_out, st)
            rec["model"].append(lg[:, 0, 0])
            rec["st"] = st
            return lg
        orc.forward_depformer = recording
        try:
            toks = orc.depformer_step(text, tout[:, None], logits_out=guided).T
        finally:
            del orc.forward_depformer
        st = rec["st"]
        din = torch.stack([tr.linear(tout, sd[f"depformer_in.{k}.weight"]) for k in range(CFG.dep_q)], dim=1)
        got = dict(din=din, k=[ls.k for ls in st.layers], v=[ls.v for ls in st.layers], logits=torch.stack(rec["model"]))
        want = depformer_ref64(sd, CFG, tout, text.repeat(2), toks.repeat(1, 2))
        out.append((tout, text, toks, got, torch.stack([x[:, 0, 0] for x in guided]), want))
    return out


def test_cfg_oracle_passes_every_checkpoint_of_both_halves(cfg_frames):
    need = {}
    for _, _, toks, got, guided, want in cfg_frames:
        for kind, k, layer, g, w in dep_checkpoints(got, want):
            r = dep_row_ratios(g, w, kind, layer)
            assert not (r > 1).any(), (kind, k, layer, r)
        for k in range(CFG.dep_q):
            # the step's guided logits are the reference's three bf16 operations on its own model logits
            assert torch.equal(guided[k], cfg_guide_bf16(got["logits"][k], B, COEF)), k
            # its tokens are the reference's guided tokens, unless the decision is within the guided logits' difference
            ref = cfg_guide64(want["logits"][k], B, COEF)
            need["guided"] = max(need.get("guided", 0.0), c_needed(guided[k], ref))
            for b in range(B):
                tol = float((guided[k][b].double() - ref[b]).abs().max()) + 1e-6
                _, unexcused = greedy_unexcused(toks[k][b:b + 1], ref[b:b + 1].argmax(-1), ref[b:b + 1].float(), tol)
                assert not unexcused, (k, b)
    _kinds_needed([(None, None, None, got, want) for _, _, _, got, _, want in cfg_frames], need)
    print(f"CFG {COEF}, 2B = {2 * B} rows: c the bf16 oracle needs " + ", ".join(f"{k} {v:.4f}" for k, v in need.items()))
    print(f"c used: din {DEP_C_DIN}, kv {[dep_c_kv(l) for l in range(CFG.depformer_num_layers)]}, logits {DEP_C_LOGITS}, "
          "guided logits exact against cfg_guide_bf16 of the model logits")


def _cfg_swapped(model, k):
    return cfg_guide_bf16(torch.cat([model[k][B:], model[k][:B]]), B, COEF)


def _cfg_null_of_previous_step(model, k):
    return cfg_guide_bf16(torch.cat([model[k][:B], model[k - 1][B:]]), B, COEF)


CFG_MUTANTS = {
    # name: (what the mutant changes, (checkpoint kind, sub-step, layer), rows that must reject it)
    "null rows fed the conditioned rows' transformer_out": ("tout", ("din", 0, None), "null"),
    "null rows given another row's previous token": ("prev", ("k", 0, 0), "null"),
    "combination with the halves swapped": (_cfg_swapped, ("guided", K, None), "guided"),
    "null logits of the previous sub-step": (_cfg_null_of_previous_step, ("guided", K, None), "guided"),
}


@pytest.mark.parametrize("name", list(CFG_MUTANTS))
def test_cfg_mutant_rejected_at_its_checkpoint_in_every_row(sd, cfg_frames, name):
    what, (kind, k, layer), rows = CFG_MUTANTS[name]
    tout, text, toks, got, guided, want = cfg_frames[0]
    if kind == "guided":            # the guided logits are held bit for bit to cfg_guide_bf16 of the model logits
        r = exact_row_ratios(what(got["logits"], k), guided[k])
    else:
        if what == "tout":
            bad = depformer_ref64(sd, CFG, torch.cat([tout[:B], tout[:B]]), text.repeat(2), toks.repeat(1, 2))
        else:
            assert (text != text.roll(-1)).all()           # else the mutant computes the right frame for that row
            mut = {"prev": lambda kk, t: torch.cat([t[kk][:B], t[kk][:B].roll(-1)])}
            bad = depformer_ref64(sd, CFG, tout, text.repeat(2), toks.repeat(1, 2), mut)
        g = {n: [t.bfloat16() for t in v] if isinstance(v, list) else v.bfloat16() for n, v in bad.items()}
        cps = {(kd, kk, ll): (gg, w) for kd, kk, ll, gg, w in dep_checkpoints(g, want)}
        r = dep_row_ratios(*cps[(kind, k, layer)], kind, layer)[B:]
    print(f"{name}: rejected at {kind} sub-step {k}{'' if layer is None else f' layer {layer}'} in the {rows} rows, "
          f"row ratios {[round(float(x), 2) for x in r]}")
    assert (r > 1).all(), (name, r)
