"""CPU: the fp64 depformer reference and the acceptance rule of tests/test_gpu_zz_depformer_ref.py, at the 7B depformer shapes.

``depformer_ref64`` restates one frame of the depformer in float64 with the bf16 model's cast points.  Two things are shown here:

* The rule accepts a correct bf16 depformer: the bf16 oracle (oracle/lm.py, fp32 accumulation in torch's order) passes at every
  checkpoint of two frames.  The constants of the rule (tests/util.py DEP_C_*) are about twice what the oracle needs.
* The rule rejects depformers with a bug that leaves the greedy tokens mostly intact: each mutant below computes a subtly wrong
  frame, and the checkpoint named beside it must reject it in every batch row.  The mutants sit at sub-step 3 and layer 2 of 6
  unless said otherwise, so that keys before and after the newest one exist and the error has layers to cross.

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
"""
import dataclasses

import pytest
import torch

from moshi_b200.config import LMConfig
from moshi_b200.synth import iter_synth_lm_tensors
from oracle import transformer as tr
from oracle.lm import LMOracle, LMSpec, scaled_embedding
from tests.util import (DEP_C_DIN, DEP_C_LOGITS, c_needed, dep_c_kv, dep_checkpoints, dep_row_ratios, depformer_ref64)

# the 7B depformer (dd 1024, 16 heads, ffn 2816, 6 layers, dep_q 8, card 2048) behind a 4096-wide temporal output
CFG = LMConfig(num_layers=1, context=16)
B, FRAMES = 4, 2
K, LAYER = 3, 2          # where the mutants act


@pytest.fixture(scope="module")
def sd():
    return {k: v for k, v in iter_synth_lm_tensors(CFG, seed=21) if k.startswith(("depformer", "linears."))}


def _oracle_frame(orc: LMOracle, sd: dict, tout: torch.Tensor, text_token: torch.Tensor) -> tuple[dict, torch.Tensor]:
    """One frame of the bf16 oracle, greedy, with its per-frame cache kept: (checkpoints in depformer_ref64's layout, the
    audio tokens [dep_q, B] it sampled)."""
    st = tr.init_state(orc.dep_spec, tout.shape[0], torch.bfloat16)
    prev, toks, logits = text_token, [], []
    for k in range(CFG.dep_q):
        lg = orc.forward_depformer(k, prev[:, None], tout[:, None], st)[:, 0, 0]
        logits.append(lg)
        prev = lg.float().argmax(-1)
        toks.append(prev)
    din = torch.stack([tr.linear(tout, sd[f"depformer_in.{k}.weight"]) for k in range(CFG.dep_q)], dim=1)
    got = dict(din=din, k=[ls.k for ls in st.layers], v=[ls.v for ls in st.layers], logits=torch.stack(logits))
    return got, torch.stack(toks)


@pytest.fixture(scope="module")
def frames(sd):
    """Per frame: (transformer_out, text token, the oracle's tokens, the oracle's checkpoints, depformer_ref64 of the frame)."""
    orc = LMOracle({**sd, "text_emb.weight": torch.zeros(1, dtype=torch.bfloat16)}, LMSpec.from_config(CFG), use_sampling=False)
    g = torch.Generator().manual_seed(5)
    out = []
    for _ in range(FRAMES):
        tout = torch.randn(B, CFG.dim, generator=g).bfloat16()
        text = torch.randint(0, CFG.text_card, (B,), generator=g)
        got, toks = _oracle_frame(orc, sd, tout, text)
        out.append((tout, text, toks, got, depformer_ref64(sd, CFG, tout, text, toks)))
    return out


def test_bf16_oracle_passes_every_checkpoint(frames):
    need = {}
    for _, _, _, got, want in frames:
        for kind, k, layer, g, w in dep_checkpoints(got, want):
            key = kind if kind in ("din", "logits") else f"kv{layer}"
            need[key] = max(need.get(key, 0.0), c_needed(g, w))
            bad = dep_row_ratios(g, w, kind, layer) > 1
            assert not bad.any(), (kind, k, layer, dep_row_ratios(g, w, kind, layer))
    print("c the bf16 oracle needs: " + ", ".join(f"{k} {v:.4f}" for k, v in need.items()))
    print(f"c used: din {DEP_C_DIN}, kv {[dep_c_kv(l) for l in range(CFG.depformer_num_layers)]}, logits {DEP_C_LOGITS}")


def test_bf16_oracle_passes_layer0_at_serving_batch(sd):
    """Layer 0's k / v at B = 256: only din, the embedding, RMSNorm and in_proj precede them, so their rare rounding flips are
    sampled here over as many rows as the fused kernel serves (the oracle's own ops, against depformer_ref64 restricted to
    layer 0, random tokens)."""
    Bs = 256
    g = torch.Generator().manual_seed(7)
    need = 0.0
    for _ in range(FRAMES):
        tout = torch.randn(Bs, CFG.dim, generator=g).bfloat16()
        text = torch.randint(0, CFG.text_card, (Bs,), generator=g)
        toks = torch.randint(0, CFG.card, (CFG.dep_q, Bs), generator=g)
        want = depformer_ref64(sd, dataclasses.replace(CFG, depformer_num_layers=1), tout, text, toks)
        prev = [text] + list(toks[:-1])
        for k in range(CFG.dep_q):
            emb = scaled_embedding(sd, "depformer_text_emb" if k == 0 else f"depformer_emb.{k - 1}", prev[k])
            x = tr.linear(tout, sd[f"depformer_in.{k}.weight"]) + emb
            xn = tr.apply_norm("rms_norm_f32", x[:, None], sd, "depformer.layers.0.norm1")[:, 0]
            qkv = tr.linear(xn, sd[f"depformer.layers.0.self_attn.in_projs.{k}.weight"]).view(Bs, 3, CFG.depformer_num_heads, 64)
            for i, kind in ((1, "k"), (2, "v")):
                w = want[kind][0][:, :, k]
                need = max(need, c_needed(qkv[:, i], w))
                assert not (dep_row_ratios(qkv[:, i], w, kind, 0) > 1).any(), (kind, k)
    print(f"layer 0 at B = {Bs}: c the bf16 oracle needs {need:.4f}, c used {dep_c_kv(0)}")


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
