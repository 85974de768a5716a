"""Seeded synthetic checkpoints with the reference's state-dict key names.

There are no real weights in the build/bench environment (no network), so parity tests, the golden
fixture generator and both bench arms use these.  Key names and tensor shapes follow what
``loaders.get_mimi(None)`` / ``LMModel(**cfg)`` produce in the reference (SURVEY.md appendix A;
``moshi/moshi/models/loaders.py:323-361``, ``lm.py:140-252``), so the same dict loads into the
reference modules (``load_state_dict``), into the CPU oracle and into the GPU handles.

Values are drawn from a ``torch.Generator`` on the requested device.  Parity work always draws on
the CPU (bit-reproducible across machines for a given torch build) and copies; the 7B bench draws on
the GPU because only timing matters there.
"""
from __future__ import annotations

import math
import typing as tp

import torch

from .config import LMConfig, MimiConfig

# Scale of the synthetic codebook entries per RVQ level, as a fraction of the level-0 residual
# standard deviation (the input-projected latent).  Level l of a residual quantizer sees a
# residual that shrinks slowly with l; the values only need to keep the nearest-code search
# input-dependent (diverse codes), they are not a model of trained codebooks.
_CODEBOOK_REL_STD = 0.35


def _uniform(gen: torch.Generator, shape, bound: float, device, dtype=torch.float32) -> torch.Tensor:
    t = torch.empty(shape, device=device, dtype=torch.float32)
    t.uniform_(-bound, bound, generator=gen)
    return t.to(dtype)


def _gen(seed: int, device) -> torch.Generator:
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return g


# ----------------------------------------------------------------------------------------------
# Mimi
# ----------------------------------------------------------------------------------------------

def seanet_layout(cfg: MimiConfig) -> tp.Tuple[list, list]:
    """Module list of the SEANet encoder / decoder as (kind, index, cin, cout, k, stride, dilation).

    Restates the construction order of ``seanet.py:170-236`` (encoder) and ``seanet.py:323-388``
    (decoder); ``index`` is the position inside the reference ``nn.Sequential`` and therefore part
    of the state-dict key.
    """
    enc = []
    mult = 1
    idx = 0
    enc.append(("conv", idx, cfg.channels, mult * cfg.n_filters, cfg.kernel_size, 1, 1))
    idx += 1
    for ratio in reversed(cfg.ratios):
        for j in range(cfg.n_residual_layers):
            enc.append(("res", idx, mult * cfg.n_filters, mult * cfg.n_filters,
                        cfg.residual_kernel_size, 1, cfg.dilation_base ** j))
            idx += 1
        idx += 1  # ELU
        enc.append(("conv", idx, mult * cfg.n_filters, mult * cfg.n_filters * 2, 2 * ratio, ratio, 1))
        idx += 1
        mult *= 2
    idx += 1  # ELU
    enc.append(("conv", idx, mult * cfg.n_filters, cfg.dimension, cfg.last_kernel_size, 1, 1))

    dec = []
    mult = 2 ** len(cfg.ratios)
    idx = 0
    dec.append(("conv", idx, cfg.dimension, mult * cfg.n_filters, cfg.kernel_size, 1, 1))
    idx += 1
    for ratio in cfg.ratios:
        idx += 1  # ELU
        dec.append(("convtr", idx, mult * cfg.n_filters, mult * cfg.n_filters // 2, 2 * ratio, ratio, 1))
        idx += 1
        for j in range(cfg.n_residual_layers):
            dec.append(("res", idx, mult * cfg.n_filters // 2, mult * cfg.n_filters // 2,
                        cfg.residual_kernel_size, 1, cfg.dilation_base ** j))
            idx += 1
        mult //= 2
    idx += 1  # ELU
    dec.append(("conv", idx, cfg.n_filters, cfg.channels, cfg.last_kernel_size, 1, 1))
    return enc, dec


def synth_mimi_state_dict(cfg: MimiConfig | None = None, seed: int = 1234,
                          device: str | torch.device = "cpu",
                          latent_std: float = 1.0) -> dict[str, torch.Tensor]:
    """Random Mimi checkpoint (fp32).  ``latent_std`` scales the codebooks (see module docstring)."""
    cfg = cfg or MimiConfig()
    g = _gen(seed, device)
    sd: dict[str, torch.Tensor] = {}

    def conv(prefix: str, cout: int, cin_per_group: int, k: int, bias: bool = True, gain: float = 1.0):
        fan_in = cin_per_group * k
        sd[prefix + ".weight"] = _uniform(g, (cout, cin_per_group, k), gain * math.sqrt(3.0 / fan_in), device)
        if bias:
            sd[prefix + ".bias"] = _uniform(g, (cout,), 0.05, device)

    def convtr(prefix: str, cin: int, cout: int, k: int, stride: int):
        # each output sample receives k/stride taps per input channel
        fan_in = cin * (k // stride)
        sd[prefix + ".weight"] = _uniform(g, (cin, cout, k), math.sqrt(3.0 / fan_in), device)
        sd[prefix + ".bias"] = _uniform(g, (cout,), 0.05, device)

    enc, dec = seanet_layout(cfg)
    for name, layers in (("encoder", enc), ("decoder", dec)):
        for kind, idx, cin, cout, k, stride, dil in layers:
            base = f"{name}.model.{idx}"
            if kind == "conv":
                conv(base + ".conv.conv", cout, cin, k, gain=1.3)
            elif kind == "convtr":
                convtr(base + ".convtr.convtr", cin, cout, k, stride)
            else:
                hidden = cin // cfg.compress
                conv(base + ".block.1.conv.conv", hidden, cin, k, gain=1.3)
                conv(base + ".block.3.conv.conv", cout, hidden, 1, gain=0.7)

    d, ff = cfg.tr_d_model, cfg.tr_dim_feedforward
    for name in ("encoder_transformer", "decoder_transformer"):
        for layer in range(cfg.tr_num_layers):
            p = f"{name}.transformer.layers.{layer}"
            sd[p + ".self_attn.in_projs.0.weight"] = _uniform(g, (3 * d, d), math.sqrt(3.0 / d), device)
            sd[p + ".self_attn.out_projs.0.weight"] = _uniform(g, (d, d), math.sqrt(3.0 / d), device)
            for n in ("norm1", "norm2"):
                sd[f"{p}.{n}.weight"] = 1.0 + _uniform(g, (d,), 0.1, device)
                sd[f"{p}.{n}.bias"] = _uniform(g, (d,), 0.05, device)
            sd[p + ".linear1.weight"] = _uniform(g, (ff, d), math.sqrt(3.0 / d), device)
            sd[p + ".linear2.weight"] = _uniform(g, (d, ff), math.sqrt(3.0 / ff), device)
            # larger than the 0.01 init so that the transformer branch matters numerically
            sd[p + ".layer_scale_1.scale"] = 0.2 + _uniform(g, (d,), 0.05, device)
            sd[p + ".layer_scale_2.scale"] = 0.2 + _uniform(g, (d,), 0.05, device)

    qd, bins = cfg.q_dimension, cfg.q_bins
    for name, n_levels in (("rvq_first", cfg.q_n_semantic), ("rvq_rest", cfg.q_n_q - cfg.q_n_semantic)):
        p = f"quantizer.{name}"
        sd[p + ".input_proj.weight"] = _uniform(g, (qd, cfg.dimension, 1), math.sqrt(3.0 / cfg.dimension), device)
        sd[p + ".output_proj.weight"] = _uniform(g, (cfg.dimension, qd, 1), math.sqrt(3.0 / qd), device)
        for level in range(n_levels):
            c = f"{p}.vq.layers.{level}._codebook"
            usage = 0.5 + torch.empty(bins, device=device).uniform_(0.0, 1.0, generator=g)
            centroids = torch.empty(bins, qd, device=device).normal_(0.0, 1.0, generator=g)
            centroids *= _CODEBOOK_REL_STD * latent_std * (0.97 ** level)
            sd[c + "._initialized"] = torch.ones(1, device=device)
            sd[c + ".cluster_usage"] = usage
            # the reference derives centroids as embedding_sum / clamp(cluster_usage, eps), core_vq.py:181-183
            sd[c + ".embedding_sum"] = centroids * usage[:, None]

    s = cfg.resample_stride
    sd["downsample.conv.conv.conv.weight"] = _uniform(
        g, (cfg.dimension, cfg.dimension, 2 * s), math.sqrt(3.0 / (cfg.dimension * 2 * s)), device)
    sd["upsample.convtr.convtr.convtr.weight"] = 0.5 + _uniform(g, (cfg.dimension, 1, 2 * s), 0.25, device)
    return sd


# ----------------------------------------------------------------------------------------------
# Moshi LM
# ----------------------------------------------------------------------------------------------

def lm_tensor_specs(cfg: LMConfig) -> list[tuple[str, tuple[int, ...], float]]:
    """(key, shape, fan_in) for every tensor of ``LMModel(**cfg)`` (SURVEY.md appendix A)."""
    specs: list[tuple[str, tuple[int, ...], float]] = []
    d, dd = cfg.dim, cfg.depformer_dim
    h, hd = cfg.ffn_hidden, cfg.depformer_ffn_hidden
    for k in range(cfg.n_q):
        specs.append((f"emb.{k}.weight", (cfg.card + 1, d), d))
    specs.append(("text_emb.weight", (cfg.text_card + 1, d), d))
    specs.append(("text_linear.weight", (cfg.text_card, d), d))
    specs.append(("out_norm.alpha", (1, 1, d), 0))
    for layer in range(cfg.num_layers):
        p = f"transformer.layers.{layer}"
        specs.append((p + ".self_attn.in_projs.0.weight", (3 * d, d), d))
        specs.append((p + ".self_attn.out_projs.0.weight", (d, d), d))
        specs.append((p + ".norm1.alpha", (1, 1, d), 0))
        specs.append((p + ".norm2.alpha", (1, 1, d), 0))
        specs.append((p + ".gating.linear_in.weight", (2 * h, d), d))
        specs.append((p + ".gating.linear_out.weight", (d, h), h))
        if cfg.cross_attention:                                      # transformer.py:727-732, 495-505
            specs.append((p + ".cross_attention.in_projs.0.weight", (3 * d, d), d))
            specs.append((p + ".cross_attention.out_projs.0.weight", (d, d), d))
            specs.append((p + ".norm_cross.weight", (d,), 0))
            specs.append((p + ".norm_cross.bias", (d,), -1))
    for i in range(cfg.extra_heads_num_heads):                       # lm.py:224-226
        specs.append((f"extra_heads.{i}.weight", (cfg.extra_heads_dim, d), d))
    for name, c in (cfg.conditioners or {}).items():                 # conditioners/text.py:106-134, base.py:105-129
        p = f"condition_provider.conditioners.{name}"
        if c["type"] == "tensor":                                    # conditioners/tensors.py: output_proj + learnt padding only
            specs.append((p + ".output_proj.weight", (d, c["tensor"]["dim"]), c["tensor"]["dim"]))
            specs.append((p + ".learnt_padding", (1, 1, d), 75.0))
            continue
        lut = c["lut"]
        specs.append((p + ".embed.weight", (lut["n_bins"] + 1, lut["dim"]), 3.0))
        specs.append((p + ".output_proj.weight", (d, lut["dim"]), lut["dim"]))
        specs.append((p + ".learnt_padding", (1, 1, d), 75.0))
    if cfg.dep_q == 0:                                               # lm.py:219-222: no depformer at all
        return specs
    n_sets, r = cfg.depformer_n_sets, cfg.depformer_low_rank_embeddings
    for k in range(n_sets):
        specs.append((f"depformer_in.{k}.weight", (dd, d), d))
    for k in range(cfg.dep_q - 1):
        specs.append((f"depformer_emb.{k}.weight", (cfg.card + 1, r or dd), r or dd))
        if r:                                                        # lm_utils.py:80-94: nn.Linear(r, dd, bias=False)
            specs.append((f"depformer_emb.{k}.low_rank.weight", (dd, r), r))
    specs.append(("depformer_text_emb.weight", (cfg.text_card + 1, r or dd), r or dd))
    if r:
        specs.append(("depformer_text_emb.low_rank.weight", (dd, r), r))
    for layer in range(cfg.depformer_num_layers):
        p = f"depformer.layers.{layer}"
        for k in range(n_sets):
            specs.append((f"{p}.self_attn.in_projs.{k}.weight", (3 * dd, dd), dd))
            specs.append((f"{p}.self_attn.out_projs.{k}.weight", (dd, dd), dd))
            specs.append((f"{p}.gating.{k}.linear_in.weight", (2 * hd, dd), dd))
            specs.append((f"{p}.gating.{k}.linear_out.weight", (dd, hd), hd))
        specs.append((p + ".norm1.alpha", (1, 1, dd), 0))
        specs.append((p + ".norm2.alpha", (1, 1, dd), 0))
    for k in range(cfg.dep_q):
        specs.append((f"linears.{k}.weight", (cfg.card, dd), dd))
    return specs


def iter_synth_lm_tensors(cfg: LMConfig, seed: int = 4242, device: str | torch.device = "cpu",
                          dtype: torch.dtype = torch.bfloat16
                          ) -> tp.Iterator[tuple[str, torch.Tensor]]:
    """Yields (key, tensor) one at a time so that a 7B model never needs two copies in memory."""
    g = _gen(seed, device)
    for key, shape, fan_in in lm_tensor_specs(cfg):
        if fan_in == 0:  # RMSNorm alpha / LayerNorm weight
            t = (1.0 + _uniform(g, shape, 0.1, device)).to(dtype)
        elif fan_in < 0:  # LayerNorm bias
            t = _uniform(g, shape, 0.05, device).to(dtype)
        else:
            # same variance as the reference's trunc-normal(std = 1/sqrt(fan_in)) init, lm_utils.py:44-56
            bound = math.sqrt(3.0 / fan_in)
            if ".out_projs." in key or "linear_out" in key:
                bound *= 0.5  # keeps the bf16 residual stream O(1) over 32 layers
            t = torch.empty(shape, device=device, dtype=dtype)
            t.uniform_(-bound, bound, generator=g)
        yield key, t


def synth_lm_state_dict(cfg: LMConfig, seed: int = 4242, device: str | torch.device = "cpu",
                        dtype: torch.dtype = torch.bfloat16) -> dict[str, torch.Tensor]:
    return dict(iter_synth_lm_tensors(cfg, seed, device, dtype))


def tiled_lm_state_dict(cfg: LMConfig, seed: int = 7, block_elems: int = 1 << 25) -> dict[str, torch.Tensor]:
    """A full-size (7.7 B parameter) bf16 checkpoint on the CPU in seconds: every tensor is cut from one seeded random block
    of ``block_elems`` values, scaled like ``iter_synth_lm_tensors`` scales it (uniform with the variance of the reference's
    init, lm_utils.py:44-56; output projections halved so that the bf16 residual stream stays O(1) over 32 layers).  Drawing 7.7 G
    independent values on the CPU takes minutes; parity and timing only need realistic, seed-reproducible values.  The same
    dict loads into the CPU oracle and into ``LMModel`` (bench.py's CPU arm, tests/test_gpu_zt_7b_parity.py)."""
    g = torch.Generator().manual_seed(seed)
    unit = (2 * torch.rand(block_elems, generator=g) - 1)              # uniform(-1, 1), fp32
    cache: dict[float, torch.Tensor] = {}
    sd: dict[str, torch.Tensor] = {}
    start = 0
    for key, shape, fan_in in lm_tensor_specs(cfg):
        n = 1
        for s_ in shape:
            n *= s_
        if fan_in == 0:
            sd[key] = (1.0 + 0.1 * unit[:n]).to(torch.bfloat16).view(shape)
            continue
        if fan_in < 0:
            sd[key] = (0.05 * unit[:n]).to(torch.bfloat16).view(shape)
            continue
        bound = math.sqrt(3.0 / fan_in)
        if ".out_projs." in key or "linear_out" in key:
            bound *= 0.5
        blk = cache.get(bound)
        if blk is None:
            blk = cache[bound] = (unit * bound).to(torch.bfloat16)
        t = torch.empty(n, dtype=torch.bfloat16)
        # successive tensors start at different offsets of the block, so that equal-shaped tensors (the 32 layers) differ
        o = 0
        while o < n:
            m = min(block_elems - start, n - o)
            t[o:o + m] = blk[start:start + m]
            o += m
            start = (start + m) % block_elems
        start = (start + 9973) % block_elems
        sd[key] = t.view(shape)
    return sd
