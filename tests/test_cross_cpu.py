"""CPU: cross-attention conditioning (the TTS models' LM) without a GPU.  The oracle restatement (tests/cross_oracle.py)
reproduces the reference's tokens and text logits bit for bit in every mode of tests/golden/lm_tiny_cross (greedy, sampled,
classifier-free guidance, a masked condition position, a mid-stream per-row memory replacement and reset, the ring wrap;
with and without cross_attention_pos_emb); the host-side conditioners and fuser equal the reference's tensors; the
configurations and fusers this path accepts and refuses."""
from __future__ import annotations

import json
from pathlib import Path

import pytest
import torch
from safetensors.torch import load_file

from moshi_b200.conditioners import ConditionAttributes, ConditionFuser, TensorCondition, build_conditioning
from moshi_b200.config import LMConfig, tiny_lm_config
from moshi_b200.models.state_dict import normalize_lm_state_dict
from moshi_b200.synth import lm_tensor_specs, synth_lm_state_dict
from oracle import scenarios
from oracle.lm import LMSpec
from tests.cross_oracle import CrossLMOracle

GOLDEN = Path(__file__).resolve().parent / "golden"
COND = {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 64}}}


@pytest.fixture(scope="module")
def gold():
    return load_file(GOLDEN / "lm_tiny_cross.safetensors"), json.loads((GOLDEN / "lm_tiny_cross.json").read_text())


def _config(info, fname):
    return tiny_lm_config(cross_attention=True, fuser=info["fusers"][fname], conditioners=COND)


def _run_oracle(g, info, fname, rname):
    cfg = _config(info, fname)
    run = info["runs"][rname]
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    name = f"{fname}.{rname}"
    orc = CrossLMOracle(sd, LMSpec.from_config(cfg), condition_cross=g[name + ".condition_cross"].clone(),
                        use_sampling=run["use_sampling"], cfg_coef=run["cfg_coef"])
    B, codes = info["B"], g[f"{fname}.codes"]
    torch.manual_seed(info["noise_seed"])
    orc.streaming(B)
    toks, logits = [], []
    for i in range(info["steps"]):
        if i == info["reset_step"]:
            orc.set_condition_cross(g[name + ".swap_cross"], [info["swap_row"]])
            mask = torch.zeros(B, dtype=torch.bool)
            mask[info["swap_row"]] = True
            orc.reset_streaming(mask)
        dbg: dict = {}
        out = orc.step(codes[i], debug=dbg)
        toks.append(torch.full((B, cfg.dep_q + 1, 1), info["none_marker"], dtype=torch.long) if out is None else out)
        logits.append(dbg["text_logits"][:, 0, 0])
    return torch.stack(toks), torch.stack(logits)


@pytest.mark.parametrize("fname", ["cross", "cross_pos"])
@pytest.mark.parametrize("rname", ["greedy", "sampled", "cfg"])
@torch.no_grad()
def test_oracle_reproduces_reference(gold, fname, rname):
    g, info = gold
    assert info["modes"][f"{fname}.{rname}"]["oracle_bit_exact_tokens"]
    toks, logits = _run_oracle(g, info, fname, rname)
    assert torch.equal(toks, g[f"{fname}.{rname}.tokens"])
    assert torch.equal(logits, g[f"{fname}.{rname}.text_logits"])
    # the swap and the masked position change the run: the fixture is not trivially insensitive to them
    assert (toks[:, :, 1:] >= 0).any()


@pytest.mark.parametrize("fname", ["cross", "cross_pos"])
@pytest.mark.parametrize("rname", ["greedy", "cfg"])
@torch.no_grad()
def test_tensor_conditioner_and_get_cross_equal_reference(gold, fname, rname):
    g, info = gold
    cfg = _config(info, fname)
    prefix = f"{fname}.condition_provider."
    weights = {k[len(fname) + 1:]: v for k, v in g.items() if k.startswith(prefix)}
    provider, fuser = build_conditioning(cfg.conditioners, cfg.fuser, cfg.dim, weights, "cpu", cross_attention=True)
    B = info["B"]
    voices = [g[f"voice.{b}"] for b in range(B)]
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(v)}) for v in voices]
    if info["runs"][rname]["cfg_coef"] != 1.0:          # the null half: nulled attributes
        attrs += [ConditionAttributes(tensor={"speaker_wavs": TensorCondition(torch.zeros_like(v), torch.zeros(1, v.shape[1], dtype=torch.bool))})
                  for v in voices]
    ct = provider(provider.prepare(attrs))
    name = f"{fname}.{rname}"
    assert torch.equal(ct["speaker_wavs"].condition, g[name + ".condition"])
    assert torch.equal(ct["speaker_wavs"].mask.to(torch.uint8), g[name + ".mask"])
    assert not bool(g[name + ".mask"][info["swap_row"]].all())      # the shorter row has learnt-padding positions
    assert torch.equal(fuser.get_cross(ct).to(torch.bfloat16), g[name + ".condition_cross"])
    swap = provider(provider.prepare([ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(g["voice.swap"])})]))
    assert torch.equal(fuser.get_cross(swap).to(torch.bfloat16), g[name + ".swap_cross"])


def test_config_accepts_cross_and_keeps_refusals():
    d = LMConfig().to_reference_kwargs()
    fuser = {"cross": ["speaker_wavs"], "cross_attention_pos_emb": True, "cross_attention_pos_emb_scale": 1.0}
    c = LMConfig.from_dict({**d, "cross_attention": True, "conditioners": COND, "fuser": fuser})
    assert c.cross_attention and "cross_attention" in c.to_reference_kwargs()
    with pytest.raises(ValueError):                     # fuser.cross without cross-attention layers
        LMConfig.from_dict({**d, "conditioners": COND, "fuser": fuser})
    with pytest.raises(ValueError):                     # a tensor conditioner no cross fuser consumes
        LMConfig.from_dict({**d, "cross_attention": True, "conditioners": COND})
    with pytest.raises(ValueError):
        LMConfig.from_dict({**d, "cross_attention": True, "conditioners": COND, "fuser": {"cross": [], "prepend": ["speaker_wavs"]}})
    with pytest.raises(ValueError):                     # the reference's cross-attention needs an nn.Linear in_proj
        LMConfig.from_dict({**d, "cross_attention": True, "quantize": True, "conditioners": COND, "fuser": fuser})
    with pytest.raises(ValueError):
        LMConfig.from_dict({**d, "cross_attention": True, "conditioners": {"x": {"type": "wav", "wav": {}}}, "fuser": {"cross": ["x"]}})


def test_fuser_needs_cross_layers():
    with pytest.raises(ValueError):
        ConditionFuser({"cross": ["speaker_wavs"]})
    with pytest.raises(ValueError):
        ConditionFuser({"prepend": ["speaker_wavs"]}, cross_attention=True)
    f = ConditionFuser({"cross": ["a", "b"]}, cross_attention=True)
    a, b = torch.randn(2, 3, 8), torch.randn(2, 4, 8)
    m = torch.ones(2, 3, dtype=torch.bool)
    assert torch.equal(f.get_cross({"a": (a, m), "b": (b, m)}), torch.cat([a, b], dim=1))
    assert f.get_sum({"a": (a, m)}) is None and f.has_conditions


def test_synth_specs_only_grow_with_cross_attention():
    plain = tiny_lm_config()
    cross = tiny_lm_config(cross_attention=True, conditioners=COND, fuser={"cross": ["speaker_wavs"]})
    base = [k for k, _, _ in lm_tensor_specs(plain)]
    extra = [k for k, _, _ in lm_tensor_specs(cross) if k not in base]
    assert [k for k, _, _ in lm_tensor_specs(cross) if k in base] == base
    L = plain.num_layers
    assert sorted(extra) == sorted([f"transformer.layers.{i}.{n}" for i in range(L) for n in (
        "cross_attention.in_projs.0.weight", "cross_attention.out_projs.0.weight", "norm_cross.weight", "norm_cross.bias")]
        + ["condition_provider.conditioners.speaker_wavs.output_proj.weight", "condition_provider.conditioners.speaker_wavs.learnt_padding"])


def test_legacy_cross_attention_names_are_split():
    w_in, w_out = torch.randn(12, 4), torch.randn(4, 4)
    out = normalize_lm_state_dict({"transformer.layers.0.cross_attention.in_proj_weight": w_in,
                                   "transformer.layers.0.cross_attention.out_proj.weight": w_out})
    assert set(out) == {"transformer.layers.0.cross_attention.in_projs.0.weight", "transformer.layers.0.cross_attention.out_projs.0.weight"}
    assert torch.equal(out["transformer.layers.0.cross_attention.in_projs.0.weight"], w_in)
