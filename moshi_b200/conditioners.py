"""Per-session conditioning in front of ``LMGen`` for the configurations that carry it (``configs/moshi_dev_2b.json``:
one LUT conditioner, fused by ``sum``).

Reference: ``moshi/moshi/conditioners/base.py:25-30`` (``ConditionType``), ``:56-88`` (``ConditionAttributes``),
``:93-168`` (``BaseConditioner.forward``: embed -> ``output_proj`` -> learnt padding where the mask is off), ``:175-351``
(``ConditionProvider``), ``:354-436`` (``ConditionFuser.get_sum``); ``conditioners/text.py:62-134`` (``NoopTokenizer``,
``LUTConditioner``); wiring ``models/loaders.py:449-487``.

Evaluating the conditioners happens once per session, outside the per-frame step: it is a handful of tiny tensor ops
(one embedding row and one ``[dim x output_dim]`` product per session), done here with torch on the model's device.
What *is* on the step path is the result, ``fuser.get_sum(condition_tensors)``, which ``LMGen`` hands to the library
(``b200_lm_set_condition_sum``) and the embedding kernel adds every frame (``lm.py:398-399``).
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
class ConditionAttributes:
    """base.py:56-88: per-sample attributes; only text attributes feed LUT conditioners."""
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


class ConditionProvider:
    """base.py:175-351 restricted to text (LUT) conditioners."""

    def __init__(self, conditioners: tp.Dict[str, LUTConditioner], device):
        self.conditioners, self.device = conditioners, device

    @property
    def text_conditions(self) -> tp.List[str]:
        return list(self.conditioners)

    def prepare(self, inputs: tp.Sequence[ConditionAttributes]) -> tp.Dict[str, tp.Any]:
        assert all(isinstance(x, ConditionAttributes) for x in inputs)
        text: tp.Dict[str, list] = {k: [] for k in self.conditioners}
        for sample in inputs:
            extra = set(sample.text) - set(self.conditioners)
            assert not extra, f"Got an unexpected attribute! Expected {list(self.conditioners)}, got {sorted(extra)}"
            for name in self.conditioners:
                if name not in sample.text:
                    raise RuntimeError(f"Some conditioners did not receive an input: {{{name!r}}}")
                text[name].append(sample.text[name])
        return {name: self.conditioners[name].prepare(batch) for name, batch in text.items()}

    def __call__(self, prepared: tp.Dict[str, tp.Any]) -> ConditionTensors:
        return {name: self.conditioners[name](p) for name, p in prepared.items()}


class ConditionFuser:
    """base.py:354-436; only the ``sum`` method reaches the streaming step of this path."""
    FUSING_METHODS = ["sum", "prepend", "cross"]

    def __init__(self, fuse2cond: tp.Dict[str, tp.List[str]]):
        assert all(k in self.FUSING_METHODS for k in fuse2cond), f"Got invalid fuse method, allowed methods: {self.FUSING_METHODS}"
        self.fuse2cond = {k: list(fuse2cond.get(k, [])) for k in self.FUSING_METHODS}
        if self.fuse2cond["cross"] or self.fuse2cond["prepend"]:
            raise ValueError("cross-attention / prepend conditioning is outside the GPU hot path (SURVEY.md 8f)")

    @property
    def has_conditions(self) -> bool:
        return bool(self.fuse2cond["sum"])

    def get_sum(self, conditions: ConditionTensors) -> torch.Tensor | None:
        total = None
        for name in self.fuse2cond["sum"]:
            cond, _ = conditions[name]
            assert cond.shape[1] == 1, cond.shape
            total = cond if total is None else total + cond
        return total

    def get_cross(self, conditions: ConditionTensors) -> None:
        return None


def build_conditioning(conditioners_cfg: tp.Optional[dict], fuser_cfg: tp.Optional[dict], output_dim: int,
                       tensors: tp.Mapping[str, torch.Tensor], device) -> tuple[ConditionProvider | None, ConditionFuser | None]:
    """``loaders.get_conditioner_provider`` + ``get_condition_fuser`` (loaders.py:449-487); weights come from the checkpoint
    under ``condition_provider.conditioners.<name>.{embed.weight, output_proj.weight, learnt_padding}``."""
    if not conditioners_cfg:
        return None, None
    conds = {}
    for name, c in conditioners_cfg.items():
        kw = dict(c[c["type"]])
        conds[name] = LUTConditioner(output_dim=output_dim, **kw)
        conds[name].load(f"condition_provider.conditioners.{name}.", tensors, device)
    fuser = ConditionFuser({k: v for k, v in (fuser_cfg or {}).items() if k in ConditionFuser.FUSING_METHODS})
    return ConditionProvider(conds, device), fuser
