"""Seeded inputs and mask/reset schedules shared by the golden generator and the tests.

Any object with ``set_exec_mask`` / ``reset_streaming`` works (reference modules, the oracle, the
GPU shims): the same schedule drives all three.
"""
from __future__ import annotations

import math

import torch

MIMI_SEED = 1234
MIMI_MASK_B = 3
MIMI_MASK_FRAMES = 8
LM_SEED = 4242
LM_NOISE_SEED = 99
LM_B = 3
LM_STEPS = 30


def sine_1s() -> torch.Tensor:
    """BASELINE.json configs[0] / SURVEY.md 8(d) config 1: 0.5*sin(2*pi*440*t), 1 s at 24 kHz."""
    t = torch.arange(24000, dtype=torch.float32) / 24000
    x = 0.5 * torch.sin(2 * math.pi * 440 * t)
    return x[None, None, :23040].contiguous()


def sine_1s_full() -> torch.Tensor:
    t = torch.arange(24000, dtype=torch.float32) / 24000
    return (0.5 * torch.sin(2 * math.pi * 440 * t))[None, None]


def mimi_noise(batch: int, frames: int, seed: int = 4242) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(batch, 1, 1920 * frames, generator=g)


def mimi_mask_events(model, frame: int, batch: int) -> None:
    """Row 1 is paused for frames 3-4, row 2 is recycled (reset) before frame 6."""
    if frame == 3:
        m = torch.ones(batch, dtype=torch.bool)
        m[1] = False
        model.set_exec_mask(m)
    if frame == 5:
        model.set_exec_mask(torch.ones(batch, dtype=torch.bool))
    if frame == 6:
        r = torch.zeros(batch, dtype=torch.bool)
        r[2] = True
        model.reset_streaming(r)


def lm_input_codes(cfg, batch: int, steps: int, seed: int = 4242) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg.card, (steps, batch, cfg.n_q - cfg.dep_q, 1), generator=g)


def lm_mask_events(gen, step: int, batch: int) -> None:
    if step == 10:
        m = torch.ones(batch, dtype=torch.bool)
        m[1] = False
        gen.set_exec_mask(m)
    if step == 12:
        gen.set_exec_mask(torch.ones(batch, dtype=torch.bool))
    if step == 20:
        r = torch.zeros(batch, dtype=torch.bool)
        r[1] = True
        gen.reset_streaming(r)


def lm_noise(cfg, batch: int, top_k_text: int = 25, top_k: int = 250):
    """The Exp(1) draws of one ``LMGen.step`` in the order and shapes the reference makes them
    (sampling.py:44 via lm.py:736 and lm.py:836): [B, k_text] then dep_q x [B, k]."""
    kt = min(top_k_text, cfg.text_card)
    ka = min(top_k, cfg.card)
    nt = torch.empty(batch, kt).exponential_(1)
    na = [torch.empty(batch, ka).exponential_(1) for _ in range(cfg.dep_q)]
    return nt, na


# ---- STT-style member of the family (SURVEY.md 8f item 2): no depformer, extra heads on the temporal output -----------------
STT_SEED = 777
STT_B = 2
STT_STEPS = 14
STT_KW = dict(dim=128, text_card=200, n_q=8, dep_q=0, card=64, num_heads=1, num_layers=2, hidden_scale=4.125, context=10,
              delays=[0] * 9, extra_heads_num_heads=2, extra_heads_dim=6)


def stt_reference_kwargs() -> dict:
    """Constructor arguments of the reference's ``LMModel`` for this scenario (7B-family options, dep_q = 0)."""
    return dict(STT_KW, existing_text_padding_id=3, causal=True, layer_scale=None, max_period=10000, gating="silu",
                norm="rms_norm_f32", positional_embedding="rope", depformer_dim=64, depformer_dim_feedforward=64,
                depformer_num_heads=1, depformer_num_layers=1, depformer_layer_scale=None, depformer_multi_linear=True,
                depformer_context=8, depformer_max_period=10000, depformer_gating="silu", depformer_pos_emb="none",
                depformer_weights_per_step=True)


def stt_state_dict(seed: int = STT_SEED) -> dict:
    """Seeded bf16 weights under the reference's key names (no depformer tensors; ``extra_heads.{i}.weight``)."""
    k = STT_KW
    d = k["dim"]
    hidden = (2 * int(k["hidden_scale"] * d)) // 3
    specs = [(f"emb.{i}.weight", (k["card"] + 1, d), d) for i in range(k["n_q"])]
    specs += [("text_emb.weight", (k["text_card"] + 1, d), d), ("text_linear.weight", (k["text_card"], d), d),
              ("out_norm.alpha", (1, 1, d), 0)]
    for layer in range(k["num_layers"]):
        p = f"transformer.layers.{layer}"
        specs += [(p + ".self_attn.in_projs.0.weight", (3 * d, d), d), (p + ".self_attn.out_projs.0.weight", (d, d), d),
                  (p + ".norm1.alpha", (1, 1, d), 0), (p + ".norm2.alpha", (1, 1, d), 0),
                  (p + ".gating.linear_in.weight", (2 * hidden, d), d), (p + ".gating.linear_out.weight", (d, hidden), hidden)]
    specs += [(f"extra_heads.{i}.weight", (k["extra_heads_dim"], d), d) for i in range(k["extra_heads_num_heads"])]
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape, fan_in in specs:
        if fan_in == 0:
            sd[key] = (1.0 + 0.1 * (2 * torch.rand(shape, generator=g) - 1)).bfloat16()
        else:
            bound = math.sqrt(3.0 / fan_in)
            sd[key] = ((2 * torch.rand(shape, generator=g) - 1) * bound).bfloat16()
    return sd


def stt_spec():
    from .lm import LMSpec
    k = STT_KW
    return LMSpec(dim=k["dim"], text_card=k["text_card"], n_q=k["n_q"], dep_q=0, card=k["card"], num_heads=k["num_heads"],
                  num_layers=k["num_layers"], hidden_scale=k["hidden_scale"], context=k["context"], delays=list(k["delays"]),
                  norm="rms_norm_f32", gating="silu", positional_embedding="rope", max_period=10000.0,
                  extra_heads_num_heads=k["extra_heads_num_heads"], extra_heads_dim=k["extra_heads_dim"])


def stt_input_codes(batch: int = STT_B, steps: int = STT_STEPS, seed: int = STT_SEED) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randint(0, STT_KW["card"], (steps, batch, STT_KW["n_q"], 1), generator=g)


# ---- the 2B configuration's delay pattern (configs/moshi_dev_2b.json: acoustic delay 2) on a tiny member of the family ------
DELAY2_SEED = 31
DELAY2_B = 2
DELAY2_STEPS = 16


def delay2_config():
    from moshi_b200.config import tiny_lm_config
    return tiny_lm_config(n_q=8, dep_q=4, delays=[0, 0, 2, 2, 2, 0, 2, 1, 2])


# ---- classifier-free guidance without a conditioner (lm.py:596-604) on the tiny LM -------------------------------------------
CFG_SEED = 9
CFG_B = 2
CFG_STEPS = 14
CFG_RESET_STEP = 8
CFG_MODES = {
    "no_text": dict(cfg_coef=2.0, cfg_is_no_text=True),
    "masked_until": dict(cfg_coef=1.5, cfg_is_masked_until=[3, 6]),
    "both": dict(cfg_coef=3.0, cfg_is_no_text=True, cfg_is_masked_until=[2, 2]),
}


# ---- sampling on peaked distributions (what a trained model produces): text / audio heads of the tiny LM scaled up ----------
PEAK_GAIN = 4.0


def peaked_state_dict(cfg, seed: int = LM_SEED) -> dict:
    """The tiny LM's seeded weights with ``text_linear`` and ``linears.*`` multiplied by PEAK_GAIN: logits of std ~4 instead
    of ~1, so that a few candidates carry the probability mass and a sampled token is decided by them rather than by the
    order of 250 near-tied candidates (random-init heads give near-uniform distributions, where the rank-indexed noise of
    sampling.py:62-64 is re-dealt by any one-ulp swap)."""
    from moshi_b200.synth import synth_lm_state_dict
    sd = synth_lm_state_dict(cfg, seed=seed)
    for k in list(sd):
        if k == "text_linear.weight" or k.startswith("linears."):
            sd[k] = (sd[k].float() * PEAK_GAIN).bfloat16()
    return sd
