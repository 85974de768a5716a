"""Hyper-parameter records for the two models on the hot path.

The field names and defaults restate the reference's configuration dictionaries so that the same
JSON / dict a reference user has keeps working:

* Mimi: ``moshi/moshi/models/loaders.py:38-88`` (``_seanet_kwargs``, ``_quantizer_kwargs``,
  ``_transformer_kwargs``, ``_mimi_config``).
* Moshi LM: ``configs/moshi_7b_202409.json`` and ``loaders.py:90-119`` (``_lm_kwargs``).

Only the options the 7B / Mimi hot path uses are honoured by the CUDA path; anything else raises
at construction time instead of silently computing something different.
"""
from __future__ import annotations

import dataclasses
import json
import typing as tp
from dataclasses import dataclass, field


@dataclass
class MimiConfig:
    sample_rate: int = 24000
    frame_rate: float = 12.5
    channels: int = 1
    # SEANet (loaders.py:38-58)
    dimension: int = 512
    n_filters: int = 64
    n_residual_layers: int = 1
    ratios: tp.List[int] = field(default_factory=lambda: [8, 6, 5, 4])  # decoder order
    kernel_size: int = 7
    residual_kernel_size: int = 3
    last_kernel_size: int = 3
    dilation_base: int = 2
    compress: int = 2
    # transformer bottlenecks (loaders.py:65-80)
    tr_d_model: int = 512
    tr_num_heads: int = 8
    tr_num_layers: int = 8
    tr_dim_feedforward: int = 2048
    tr_context: int = 250
    tr_max_period: float = 10000.0
    tr_layer_scale: float = 0.01
    # quantizer (loaders.py:59-64)
    q_dimension: int = 256
    q_bins: int = 2048
    q_n_q: int = 32          # codebooks stored in the checkpoint
    q_n_semantic: int = 1
    num_codebooks: int = 8   # codebooks active (loaders.py:323-326 default)

    @property
    def hop_length(self) -> int:
        h = 1
        for r in self.ratios:
            h *= r
        return h

    @property
    def encoder_frame_rate(self) -> float:
        return self.sample_rate / self.hop_length

    @property
    def frame_size(self) -> int:
        return int(self.sample_rate / self.frame_rate)

    @property
    def resample_stride(self) -> int:
        return int(self.encoder_frame_rate / self.frame_rate)

    @staticmethod
    def from_reference_dict(cfg: dict | None, num_codebooks: int = 8) -> "MimiConfig":
        """Accepts the nested dict layout of ``loaders._mimi_config``."""
        if cfg is None:
            return MimiConfig(num_codebooks=num_codebooks)
        sea, qt, tr = cfg["seanet"], cfg["quantizer"], cfg["transformer"]
        unsupported = []
        if sea.get("norm", "none") != "none":
            unsupported.append("seanet.norm")
        if sea.get("pad_mode", "constant") != "constant":
            unsupported.append("seanet.pad_mode")
        if not sea.get("true_skip", True):
            unsupported.append("seanet.true_skip")
        if tr.get("gating", "none") != "none" or tr.get("norm", "layer_norm") != "layer_norm":
            unsupported.append("transformer.gating/norm")
        if tr.get("positional_embedding", "rope") != "rope":
            unsupported.append("transformer.positional_embedding")
        if sea.get("activation", "ELU") != "ELU" or sea.get("activation_params", {"alpha": 1.0}).get("alpha", 1.0) != 1.0:
            unsupported.append("seanet.activation")
        if not sea.get("causal", True) or not tr.get("causal", True):
            unsupported.append("causal=False")
        if sea.get("disable_norm_outer_blocks", 0) != 0:
            unsupported.append("seanet.disable_norm_outer_blocks")
        if not tr.get("conv_layout", True):
            unsupported.append("transformer.conv_layout=False")
        if unsupported:
            raise ValueError(f"Mimi options outside the GPU hot path: {unsupported}")
        return MimiConfig(
            sample_rate=cfg["sample_rate"], frame_rate=cfg["frame_rate"], channels=cfg["channels"],
            dimension=sea["dimension"], n_filters=sea["n_filters"],
            n_residual_layers=sea["n_residual_layers"], ratios=list(sea["ratios"]),
            kernel_size=sea["kernel_size"], residual_kernel_size=sea["residual_kernel_size"],
            last_kernel_size=sea["last_kernel_size"], dilation_base=sea["dilation_base"],
            compress=sea["compress"], tr_d_model=tr["d_model"], tr_num_heads=tr["num_heads"],
            tr_num_layers=tr["num_layers"], tr_dim_feedforward=tr["dim_feedforward"],
            tr_context=tr["context"], tr_max_period=float(tr["max_period"]),
            tr_layer_scale=tr["layer_scale"], q_dimension=qt["dimension"], q_bins=qt["bins"],
            q_n_q=qt["n_q"], num_codebooks=num_codebooks)

    def to_reference_dict(self) -> dict:
        """The nested dict ``loaders.get_mimi(mimi_config=...)`` takes (used by the golden generator)."""
        seanet = {
            "channels": self.channels, "dimension": self.dimension, "causal": True,
            "n_filters": self.n_filters, "n_residual_layers": self.n_residual_layers,
            "activation": "ELU", "compress": self.compress, "dilation_base": self.dilation_base,
            "disable_norm_outer_blocks": 0, "kernel_size": self.kernel_size,
            "residual_kernel_size": self.residual_kernel_size,
            "last_kernel_size": self.last_kernel_size, "norm": "none", "pad_mode": "constant",
            "ratios": list(self.ratios), "true_skip": True,
        }
        quantizer = {"dimension": self.q_dimension, "n_q": self.q_n_q, "bins": self.q_bins,
                     "input_dimension": self.dimension, "output_dimension": self.dimension}
        transformer = {
            "d_model": self.tr_d_model, "num_heads": self.tr_num_heads,
            "num_layers": self.tr_num_layers, "causal": True, "layer_scale": self.tr_layer_scale,
            "context": self.tr_context, "conv_layout": True, "max_period": self.tr_max_period,
            "gating": "none", "norm": "layer_norm", "positional_embedding": "rope",
            "dim_feedforward": self.tr_dim_feedforward, "input_dimension": self.dimension,
            "output_dimensions": [self.dimension],
        }
        return {"sample_rate": self.sample_rate, "channels": self.channels,
                "frame_rate": self.frame_rate, "seanet": seanet, "quantizer": quantizer,
                "transformer": transformer}


@dataclass
class LMConfig:
    """``LMModel.__init__`` keyword arguments (``lm.py:76-113``) restricted to the 7B family."""
    dim: int = 4096
    text_card: int = 32000
    existing_text_padding_id: int = 3
    n_q: int = 16
    dep_q: int = 8
    card: int = 2048
    num_heads: int = 32
    num_layers: int = 32
    hidden_scale: float = 4.125
    causal: bool = True
    layer_scale: tp.Optional[float] = None
    context: int = 3000
    max_period: float = 10000.0
    gating: str = "silu"
    norm: str = "rms_norm_f32"
    positional_embedding: str = "rope"
    depformer_dim: int = 1024
    depformer_dim_feedforward: int = 4224
    depformer_num_heads: int = 16
    depformer_num_layers: int = 6
    depformer_layer_scale: tp.Optional[float] = None
    depformer_multi_linear: bool = True
    depformer_context: int = 8
    depformer_max_period: float = 10000.0
    depformer_gating: str = "silu"
    depformer_pos_emb: str = "none"
    depformer_weights_per_step: bool = True
    # lm.py:125-127, 172-181, transformer.py:291-316: sub-step k runs weight set schedule[k] of depformer_in and of every depformer
    # layer's in_projs / out_projs / gating; max(schedule) + 1 sets are stored
    depformer_weights_per_step_schedule: tp.Optional[tp.List[int]] = None
    # lm.py:186-196, lm_utils.py:80-124: each depformer embedding is a [V, r] table followed by a bias-free nn.Linear(r, depformer_dim)
    depformer_low_rank_embeddings: tp.Optional[int] = None
    quantize: bool = False       # LMModel(quantize=True), lm.py:107,242-243: every nn.Linear becomes an int8 QLinear
    extra_heads_num_heads: int = 0   # lm.py:108-109, 224-226: nn.Linear(dim, extra_heads_dim) heads on the temporal output (STT)
    extra_heads_dim: int = 6
    # lm.py:110-118 via loaders.get_conditioner_provider / get_condition_fuser (loaders.py:449-487): the JSON's "conditioners"
    # and "fuser" sections (configs/moshi_dev_2b.json).  LUT conditioners fused by "sum", and tensor conditioners fused by
    # "cross" into the temporal layers' cross-attention (cross_attention=True, the TTS models) are on the step path.
    conditioners: tp.Optional[dict] = None
    fuser: tp.Optional[dict] = None
    cross_attention: bool = False
    delays: tp.List[int] = field(
        default_factory=lambda: [0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1])

    @property
    def num_codebooks(self) -> int:
        return self.n_q + 1

    @property
    def max_delay(self) -> int:
        return max(self.delays)

    @property
    def ffn_hidden(self) -> int:
        """Gated hidden width, ``gating.py:52-58``."""
        return _gated_hidden(self.dim, int(self.hidden_scale * self.dim))

    @property
    def depformer_ffn_hidden(self) -> int:
        return _gated_hidden(self.depformer_dim, self.depformer_dim_feedforward)

    @property
    def depformer_n_sets(self) -> int:
        """Weight sets of the depformer's per-step linears (lm.py:177-178, transformer.py:399-401)."""
        s = self.depformer_weights_per_step_schedule
        return max(s) + 1 if s else self.dep_q

    @staticmethod
    def from_dict(d: dict) -> "LMConfig":
        d = dict(d)
        d.pop("depformer_causal", None)  # deprecated key, dropped by loaders.py:391-392
        known = {f.name for f in dataclasses.fields(LMConfig)}
        extra = sorted(set(d) - known)
        if extra:
            raise ValueError(f"LM options outside the GPU hot path: {extra}")
        cfg = LMConfig(**d)
        cfg.check_supported()
        return cfg

    @staticmethod
    def from_json(path: str) -> "LMConfig":
        with open(path) as f:
            return LMConfig.from_dict(json.load(f))

    def to_reference_kwargs(self) -> dict:
        """Keyword arguments of the reference's ``LMModel`` (the ``conditioners`` / ``fuser`` JSON sections are turned into
        modules by ``loaders.get_conditioner_provider`` / ``get_condition_fuser`` there, so they are not constructor arguments)."""
        d = dataclasses.asdict(self)
        d.pop("conditioners")
        d.pop("fuser")
        return d

    def check_supported(self) -> None:
        bad = []
        if self.norm != "rms_norm_f32":
            bad.append("norm")
        if self.gating != "silu" or self.depformer_gating != "silu":
            bad.append("gating")
        if self.positional_embedding != "rope" or self.depformer_pos_emb != "none":
            bad.append("positional_embedding")
        if self.layer_scale is not None or self.depformer_layer_scale is not None:
            bad.append("layer_scale")
        if not (self.depformer_multi_linear and self.depformer_weights_per_step):
            bad.append("depformer_multi_linear/weights_per_step")
        if len(self.delays) != self.n_q + 1:
            bad.append("delays")
        if not self.causal:
            bad.append("causal=False")
        if self.dep_q and self.depformer_context < self.dep_q:
            bad.append("depformer_context < dep_q (the depformer attends over all of a frame's codebooks)")
        fuser = self.fuser or {}
        if fuser.get("prepend"):
            bad.append("prepend conditioning (only fuser.sum and fuser.cross are on the step path)")
        if fuser.get("cross") and not self.cross_attention:     # the reference fails at the first step (transformer.py:786)
            bad.append("fuser.cross on a model without cross_attention")
        if self.cross_attention and self.quantize:              # _compute_cross_attention asserts an nn.Linear in_proj
            bad.append("cross_attention with quantize=True")
        for name, c in (self.conditioners or {}).items():
            if c.get("type") == "tensor":
                if name not in (fuser.get("cross") or []):
                    bad.append(f"tensor conditioner {name!r} that no fuser.cross consumes")
            elif c.get("type") != "lut":
                bad.append(f"conditioner {name!r} of type {c.get('type')!r} (only 'lut' and 'tensor')")
        if not 0 <= self.dep_q <= 16 or not 1 <= self.n_q <= 32 or self.dep_q > self.n_q:
            bad.append("n_q / dep_q (n_q <= 32, 0 <= dep_q <= 16)")
        if self.dim % self.num_heads or (self.dep_q and self.depformer_dim % self.depformer_num_heads):
            bad.append("heads")
        if self.quantize and any(k % 16 for k in (self.dim, self.ffn_hidden, self.depformer_dim, self.depformer_ffn_hidden)):
            bad.append("quantize (int8 k-extents must be multiples of 16)")
        bad += self._depformer_sharing_problems()
        if bad:
            raise ValueError(f"LM options outside the GPU hot path: {bad}")

    def _depformer_sharing_problems(self) -> list[str]:
        bad = []
        s = self.depformer_weights_per_step_schedule
        if s is not None:
            if not (self.depformer_multi_linear and self.depformer_weights_per_step):
                bad.append("depformer_weights_per_step_schedule without depformer_multi_linear and depformer_weights_per_step")
            if len(s) != self.dep_q:
                bad.append(f"depformer_weights_per_step_schedule of length {len(s)} (one entry per depformer step: {self.dep_q})")
            if any(not isinstance(j, int) or not 0 <= j < self.dep_q for j in s):
                bad.append(f"depformer_weights_per_step_schedule entries must be in [0, dep_q = {self.dep_q})")
        r = self.depformer_low_rank_embeddings
        if r is not None and (not isinstance(r, int) or not 1 <= r <= LOW_RANK_MAX):
            bad.append(f"depformer_low_rank_embeddings = {r!r} (the rank must be in [1, {LOW_RANK_MAX}]: the load-time expansion "
                       "holds one row of the factor table in shared memory)")
        return bad


# largest depformer_low_rank_embeddings the load-time table expansion takes (b200_lm_set_depformer_low_rank)
LOW_RANK_MAX = 4096


def _gated_hidden(dim: int, dim_feedforward: int) -> int:
    if dim_feedforward == 4 * dim:
        return (21 * dim) // 8
    return (2 * dim_feedforward) // 3


MOSHI_7B = LMConfig()


def tiny_lm_config(**over) -> LMConfig:
    """A scaled-down member of the 7B family that the CPU oracle steps in milliseconds."""
    base = dict(dim=256, text_card=500, n_q=16, dep_q=8, card=64, num_heads=2, num_layers=3,
                hidden_scale=4.125, context=12, depformer_dim=128, depformer_dim_feedforward=528,
                depformer_num_heads=2, depformer_num_layers=2)
    base.update(over)
    return LMConfig(**base)
