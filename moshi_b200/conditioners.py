"""Per-session conditioning in front of ``LMGen`` for the configurations that carry it (``configs/moshi_dev_2b.json``:
one LUT conditioner, fused by ``sum``; the TTS models: tensor conditioners fused by ``cross`` into the temporal layers'
cross-attention).

Reference: ``moshi/moshi/conditioners/base.py:25-30`` (``ConditionType``), ``:56-88`` (``ConditionAttributes``),
``:93-168`` (``BaseConditioner.forward``: embed -> ``output_proj`` -> learnt padding where the mask is off), ``:175-351``
(``ConditionProvider``), ``:354-436`` (``ConditionFuser.get_sum``); ``conditioners/text.py:62-134`` (``NoopTokenizer``,
``LUTConditioner``); ``conditioners/tensors.py`` (``TensorConditioner``) and ``base.py:33-59`` (``TensorCondition``),
``:392-409`` (``ConditionFuser.get_cross``); wiring ``models/loaders.py:449-487``.

Evaluating the conditioners happens once per session, outside the per-frame step: it is a handful of tiny tensor ops
(one embedding row and one ``[dim x output_dim]`` product per session), done here with torch on the model's device.
What *is* on the step path is the result, ``fuser.get_sum(condition_tensors)``, which ``LMGen`` hands to the library
(``b200_lm_set_condition_sum``) and the embedding kernel adds every frame (``lm.py:398-399``), and
``fuser.get_cross(condition_tensors)``, from which the library computes every layer's cross-attention keys and values once
per session (``b200_lm_set_condition_cross``, ``transformer.py:495-505``).
"""
from __future__ import annotations

import hashlib
import typing as tp
from dataclasses import dataclass, field

import torch


class ConditionType(tp.NamedTuple):
    """``(condition [B, T, dim], mask [B, T])`` (base.py:25-30)."""
    condition: torch.Tensor
    mask: torch.Tensor


ConditionTensors = tp.Dict[str, ConditionType]


@dataclass
class TensorCondition:
    """base.py:33-59: the input of a tensor conditioner, ``tensor`` [B | 1, T, dim] and ``mask`` [B | 1, T]."""
    tensor: torch.Tensor
    mask: torch.Tensor

    @staticmethod
    def from_tensor(tensor: torch.Tensor) -> "TensorCondition":
        B, T, _ = tensor.shape
        return TensorCondition(tensor, torch.ones(B, T, dtype=torch.bool, device=tensor.device))

    @staticmethod
    def cat(conditions: tp.Sequence["TensorCondition"]) -> "TensorCondition":
        """One row per condition, zero-padded (mask off) to the longest T."""
        assert conditions, "Cannot cat empty list."
        ref = conditions[0].tensor
        B, _, D = ref.shape
        assert B == 1
        T = max(c.tensor.shape[1] for c in conditions)
        mask = torch.zeros(len(conditions), T, dtype=torch.bool, device=ref.device)
        tensor = torch.zeros(len(conditions), T, D, dtype=ref.dtype, device=ref.device)
        for b, c in enumerate(conditions):
            tensor[b, :c.tensor.shape[1], :] = c.tensor[0]
            mask[b, :c.mask.shape[1]] = c.mask[0]
        return TensorCondition(tensor, mask)


@dataclass
class ConditionAttributes:
    """base.py:56-88: per-sample attributes; text attributes feed LUT conditioners, tensor attributes tensor conditioners."""
    text: tp.Dict[str, tp.Optional[str]] = field(default_factory=dict)
    tensor: tp.Dict[str, tp.Any] = field(default_factory=dict)


def _hash_trick(word: str, vocab_size: int) -> int:
    return int(hashlib.sha256(word.encode("utf-8")).hexdigest(), 16) % vocab_size      # text.py:35-45


class NoopTokenizer:
    """text.py:62-103: one index per whole string; ``None`` -> the padding index with an empty mask."""

    def __init__(self, n_bins: int, possible_values: tp.Optional[tp.List[str]] = None):
        self.n_bins, self.pad_idx = n_bins, n_bins
        self.possible_values = None if possible_values is None else {v: i for i, v in enumerate(possible_values)}
        if self.possible_values is not None:
            assert n_bins >= len(self.possible_values)

    def __call__(self, texts: tp.List[tp.Optional[str]]) -> tp.Tuple[torch.Tensor, torch.Tensor]:
        out, lengths = [], []
        for text in texts:
            if text is None:
                out.append(self.pad_idx)
                lengths.append(0)
                continue
            if self.possible_values is None:
                out.append(_hash_trick(text, self.n_bins))
            elif text not in self.possible_values:
                raise ValueError(f"'{text}' is not in possible_values {self.possible_values}")
            else:
                out.append(self.possible_values[text])
            lengths.append(1)
        tokens = torch.tensor(out).int()[:, None]
        lengths_t = torch.tensor(lengths)
        final = max(int(lengths_t.max().item()) if len(lengths) else 0, 1)          # text.py:18-32 length_to_mask
        mask = torch.arange(final)[None, :] < lengths_t[:, None]
        return tokens, mask


class LUTConditioner:
    """``LUTConditioner`` (text.py:106-134) on top of ``BaseConditioner.forward`` (base.py:151-168), weights given."""

    def __init__(self, n_bins: int, dim: int, output_dim: int, tokenizer: str = "noop",
                 possible_values: tp.Optional[tp.List[str]] = None, **_unused):
        if tokenizer != "noop":
            raise ValueError(f"unrecognized tokenizer `{tokenizer}`.")
        self.dim, self.output_dim = dim, output_dim
        self.tokenizer = NoopTokenizer(n_bins, possible_values)
        self.n_bins = n_bins
        self.embed_weight: torch.Tensor | None = None          # [n_bins + 1, dim]
        self.output_proj_weight: torch.Tensor | None = None    # [output_dim, dim]
        self.learnt_padding: torch.Tensor | None = None        # [1, 1, output_dim]

    def load(self, prefix: str, sd: tp.Mapping[str, torch.Tensor], device) -> None:
        self.embed_weight = sd[prefix + "embed.weight"].to(device)
        self.output_proj_weight = sd[prefix + "output_proj.weight"].to(device)
        lp = sd.get(prefix + "learnt_padding")
        self.learnt_padding = None if lp is None else lp.to(device)
        assert self.embed_weight.shape == (self.n_bins + 1, self.dim), self.embed_weight.shape
        assert self.output_proj_weight.shape == (self.output_dim, self.dim), self.output_proj_weight.shape

    def prepare(self, texts: tp.List[tp.Optional[str]]):
        tokens, mask = self.tokenizer(texts)
        dev = self.embed_weight.device
        return tokens.to(dev), mask.to(dev)

    def __call__(self, prepared) -> ConditionType:
        tokens, mask = prepared
        cond = torch.nn.functional.embedding(tokens.long(), self.embed_weight)
        cond = torch.nn.functional.linear(cond, self.output_proj_weight)
        maskf = mask.float()[..., None]
        if self.learnt_padding is not None:
            cond = cond * maskf + self.learnt_padding * (1 - maskf)
        else:
            cond = cond * maskf
        return ConditionType(cond, mask)


class TensorConditioner:
    """``TensorConditioner`` (conditioners/tensors.py) on top of ``BaseConditioner.forward`` (base.py:151-168), weights given:
    the tensor itself through ``output_proj``, learnt padding where the mask is off."""

    def __init__(self, dim: int, output_dim: int, pad_empty: bool = True, **_unused):
        self.dim, self.output_dim, self.pad_empty = dim, output_dim, pad_empty
        self.output_proj_weight: torch.Tensor | None = None    # [output_dim, dim]
        self.learnt_padding: torch.Tensor | None = None        # [1, 1, output_dim]

    def load(self, prefix: str, sd: tp.Mapping[str, torch.Tensor], device) -> None:
        # the reference's conditioner parameters are float32 whatever the LM's dtype (base.py:121-129)
        self.output_proj_weight = sd[prefix + "output_proj.weight"].to(device=device, dtype=torch.float32)
        lp = sd.get(prefix + "learnt_padding")
        self.learnt_padding = None if lp is None else lp.to(device=device, dtype=torch.float32)
        assert self.output_proj_weight.shape == (self.output_dim, self.dim), self.output_proj_weight.shape

    def prepare(self, tensor: TensorCondition) -> TensorCondition:
        dev = self.output_proj_weight.device
        return TensorCondition(tensor.tensor.to(device=dev), tensor.mask.to(device=dev))

    def __call__(self, prepared: TensorCondition) -> ConditionType:
        cond, mask = prepared.tensor, prepared.mask
        B, T, C = cond.shape
        if T == 0 and self.pad_empty:
            cond = torch.zeros(B, T, C, device=cond.device, dtype=cond.dtype)
            mask = torch.zeros_like(cond[..., 0], dtype=torch.bool)
        cond = torch.nn.functional.linear(cond, self.output_proj_weight)
        maskf = mask.float()[..., None]
        if self.learnt_padding is not None:
            cond = cond * maskf + self.learnt_padding * (1 - maskf)
        else:
            cond = cond * maskf
        return ConditionType(cond, mask)


class ConditionProvider:
    """base.py:175-351: text (LUT) and tensor conditioners."""

    def __init__(self, conditioners: tp.Dict[str, LUTConditioner | TensorConditioner], device):
        self.conditioners, self.device = conditioners, device

    @property
    def text_conditions(self) -> tp.List[str]:
        return [k for k, c in self.conditioners.items() if isinstance(c, LUTConditioner)]

    @property
    def tensor_conditions(self) -> tp.List[str]:
        return [k for k, c in self.conditioners.items() if isinstance(c, TensorConditioner)]

    def prepare(self, inputs: tp.Sequence[ConditionAttributes]) -> tp.Dict[str, tp.Any]:
        assert all(isinstance(x, ConditionAttributes) for x in inputs)
        text: tp.Dict[str, list] = {k: [] for k in self.text_conditions}
        tensors: tp.Dict[str, list] = {k: [] for k in self.tensor_conditions}
        for sample in inputs:
            extra = (set(sample.text) - set(text)) | (set(sample.tensor) - set(tensors))
            assert not extra, f"Got an unexpected attribute! Expected {list(self.conditioners)}, got {sorted(extra)}"
            for names, given, out in ((text, sample.text, text), (tensors, sample.tensor, tensors)):
                for name in names:
                    if name not in given:
                        raise RuntimeError(f"Some conditioners did not receive an input: {{{name!r}}}")
                    out[name].append(given[name])
        prepared = {name: self.conditioners[name].prepare(batch) for name, batch in text.items()}
        prepared.update({name: self.conditioners[name].prepare(TensorCondition.cat(batch)) for name, batch in tensors.items()})
        return prepared

    def __call__(self, prepared: tp.Dict[str, tp.Any]) -> ConditionTensors:
        return {name: self.conditioners[name](p) for name, p in prepared.items()}


class ConditionFuser:
    """base.py:354-436: ``sum`` and ``cross`` reach the streaming step of this path, ``cross`` only for an LM with
    cross-attention layers (``cross_attention``: the reference would fail at its first step)."""
    FUSING_METHODS = ["sum", "prepend", "cross"]

    def __init__(self, fuse2cond: tp.Dict[str, tp.List[str]], cross_attention_pos_emb: bool = False,
                 cross_attention_pos_emb_scale: float = 1.0, cross_attention: bool = False):
        assert all(k in self.FUSING_METHODS for k in fuse2cond), f"Got invalid fuse method, allowed methods: {self.FUSING_METHODS}"
        self.fuse2cond = {k: list(fuse2cond.get(k, [])) for k in self.FUSING_METHODS}
        self.cross_attention_pos_emb = cross_attention_pos_emb
        self.cross_attention_pos_emb_scale = cross_attention_pos_emb_scale
        if self.fuse2cond["prepend"]:
            raise ValueError("prepend conditioning is outside the GPU hot path (SURVEY.md 8f)")
        if self.fuse2cond["cross"] and not cross_attention:
            raise ValueError("cross conditioning needs an LM with cross-attention layers (cross_attention=True)")

    @property
    def has_conditions(self) -> bool:
        return bool(self.fuse2cond["sum"] or self.fuse2cond["cross"])

    def get_sum(self, conditions: ConditionTensors) -> torch.Tensor | None:
        total = None
        for name in self.fuse2cond["sum"]:
            cond, _ = conditions[name]
            assert cond.shape[1] == 1, cond.shape
            total = cond if total is None else total + cond
        return total

    def get_cross(self, conditions: ConditionTensors) -> torch.Tensor | None:
        """base.py:392-409: the cross conditions concatenated along T, plus the scaled sin embedding of the positions."""
        cross = None
        for name in self.fuse2cond["cross"]:
            cond, _ = conditions[name]
            cross = cond if cross is None else torch.cat([cross, cond], dim=1)
        if self.cross_attention_pos_emb and cross is not None:
            positions = torch.arange(cross.shape[1], device=cross.device).view(1, -1, 1)
            cross = cross + self.cross_attention_pos_emb_scale * _sin_embedding(positions, cross.shape[-1]).to(cross.dtype)
        return cross


def _sin_embedding(positions: torch.Tensor, dim: int, max_period: float = 10000) -> torch.Tensor:
    """``create_sin_embedding`` (transformer.py:139-165) in float32: [cos | sin] of positions / max_period ** (i / (dim/2 - 1))."""
    half = dim // 2
    positions = positions.to(torch.float32)
    adim = torch.arange(half, device=positions.device, dtype=torch.float32).view(1, 1, -1)
    mp = torch.full([], max_period, device=positions.device, dtype=torch.float32)
    phase = positions / (mp ** (adim / (half - 1)))
    return torch.cat([torch.cos(phase), torch.sin(phase)], dim=-1)


def build_conditioning(conditioners_cfg: tp.Optional[dict], fuser_cfg: tp.Optional[dict], output_dim: int,
                       tensors: tp.Mapping[str, torch.Tensor], device,
                       cross_attention: bool = False) -> tuple[ConditionProvider | None, ConditionFuser | None]:
    """``loaders.get_conditioner_provider`` + ``get_condition_fuser`` (loaders.py:449-487); weights come from the checkpoint
    under ``condition_provider.conditioners.<name>.{embed.weight, output_proj.weight, learnt_padding}``.  ``cross_attention``:
    whether the LM has cross-attention layers (``LMConfig.cross_attention``)."""
    if not conditioners_cfg:
        return None, None
    conds: tp.Dict[str, LUTConditioner | TensorConditioner] = {}
    for name, c in conditioners_cfg.items():
        kw = dict(c[c["type"]])
        conds[name] = (TensorConditioner if c["type"] == "tensor" else LUTConditioner)(output_dim=output_dim, **kw)
        conds[name].load(f"condition_provider.conditioners.{name}.", tensors, device)
    fuser_cfg = fuser_cfg or {}
    pos = {k: fuser_cfg[k] for k in ("cross_attention_pos_emb", "cross_attention_pos_emb_scale") if k in fuser_cfg}
    fuser = ConditionFuser({k: v for k, v in fuser_cfg.items() if k in ConditionFuser.FUSING_METHODS},
                           cross_attention=cross_attention, **pos)
    return ConditionProvider(conds, device), fuser
