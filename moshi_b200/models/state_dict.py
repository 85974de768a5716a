"""Checkpoint key normalisation: the on-disk names the reference accepts map to the module names.

* packed attention weights ``self_attn.in_proj_weight`` / ``in_proj.weight`` / ``out_proj.weight`` (and the same names
  under ``cross_attention.``) of shape ``[mult * rows, in]`` become ``in_projs.{i}.weight`` / ``out_projs.{i}.weight``
  (load hook ``moshi/moshi/modules/transformer.py:422-446``);
* legacy codebook buffers ``inited`` / ``cluster_size`` / ``embed_avg`` / ``embed_sum``
  become ``_initialized`` / ``cluster_usage`` / ``embedding_sum`` (``core_vq.py:162-176``);
* the Rust / candle layout of the LM (``scripts/import_rust.py``): per-step depformer slices ``depformer.<k>.*``.
"""
from __future__ import annotations

import re
import typing as tp

import torch

_CODEBOOK_RENAMES = {"inited": "_initialized", "cluster_size": "cluster_usage",
                     "embed_avg": "embedding_sum", "embed_sum": "embedding_sum"}


def _split_attention(sd: tp.Mapping[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    out: dict[str, torch.Tensor] = {}
    for key, w in sd.items():
        if key.endswith(("self_attn.in_proj_weight", "self_attn.in_proj.weight", "cross_attention.in_proj_weight",
                         "cross_attention.in_proj.weight")):
            base = key[: key.rindex("in_proj")]
            mult = max(1, w.shape[0] // (3 * w.shape[1]))
            for i, part in enumerate(w.view(mult, -1, w.shape[1])):
                out[f"{base}in_projs.{i}.weight"] = part
        elif key.endswith(("self_attn.out_proj.weight", "cross_attention.out_proj.weight")):
            base = key[: key.rindex("out_proj")]
            mult = max(1, w.shape[0] // w.shape[1])
            for i, part in enumerate(w.view(mult, -1, w.shape[1])):
                out[f"{base}out_projs.{i}.weight"] = part
        else:
            out[key] = w
    return out


def normalize_mimi_state_dict(sd: tp.Mapping[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    out = {}
    for key, v in _split_attention(sd).items():
        head, _, leaf = key.rpartition(".")
        if head.endswith("_codebook") and leaf in _CODEBOOK_RENAMES:
            key = f"{head}.{_CODEBOOK_RENAMES[leaf]}"
        out[key] = v
    return out


_CANDLE = re.compile(r"^depformer\.(\d+)\.(.+)$")


def _from_candle(sd: tp.Mapping[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """The Rust / candle checkpoint layout written by ``scripts/import_rust.py:45-113`` (what ``rust/moshi-core`` loads,
    ``lm.rs:486-635``): the temporal transformer keeps the reference's names; the depformer is stored per codebook step as
    ``depformer.<k>.{linear_in, linear_out, emb}.weight`` and ``depformer.<k>.transformer.layers.<l>.*`` (one slice of the
    per-step weights each, norms repeated).  Mapped back onto the reference's module names."""
    out: dict[str, torch.Tensor] = {}
    for key, v in sd.items():
        m = _CANDLE.match(key)
        if m is None:
            out[key] = v
            continue
        k, rest = int(m.group(1)), m.group(2)
        if rest == "linear_in.weight":
            out[f"depformer_in.{k}.weight"] = v
        elif rest == "linear_out.weight":
            out[f"linears.{k}.weight"] = v
        elif rest.startswith("emb."):
            base = "depformer_text_emb" if k == 0 else f"depformer_emb.{k - 1}"
            out[f"{base}.{rest[len('emb.'):]}"] = v
        elif rest.startswith("transformer.layers."):
            layer, leaf = rest[len("transformer.layers."):].split(".", 1)
            p = f"depformer.layers.{layer}."
            if leaf == "self_attn.in_proj_weight":
                out[p + f"self_attn.in_projs.{k}.weight"] = v
            elif leaf == "self_attn.out_proj.weight":
                out[p + f"self_attn.out_projs.{k}.weight"] = v
            elif leaf.startswith("norm"):
                if k == 0:                       # the same alpha is written under every step (import_rust.py:98-103)
                    out[p + leaf] = v
            elif leaf.startswith("gating."):
                out[p + f"gating.{k}." + leaf[len("gating."):]] = v
            else:
                raise ValueError(f"unexpected tensor {key!r} in a candle-layout checkpoint")
        else:
            raise ValueError(f"unexpected tensor {key!r} in a candle-layout checkpoint")
    return out


def candle_refusal(cfg, key: str) -> str | None:
    """Why the candle-layout tensor ``key`` cannot be loaded into an LM of configuration ``cfg`` (None: it can).
    ``scripts/import_rust.py:69-110`` writes one slice per depformer step, a weight-sharing schedule unrolled into copies of
    the shared sets: slice k holds set schedule[k], not set k, so a scheduled model would read the wrong weights from the
    renamed slices.  Low-rank depformer embeddings have no candle form that this loader knows."""
    if _CANDLE.match(key) is None:
        return None
    if cfg.cross_attention:
        return "candle-layout checkpoints of a cross-attention LM are not supported; load its safetensors checkpoint"
    if cfg.depformer_weights_per_step_schedule is not None:
        return ("candle-layout checkpoints of an LM with depformer_weights_per_step_schedule are not supported (the layout unrolls "
                "the schedule into one slice per step); load its safetensors checkpoint")
    if cfg.depformer_low_rank_embeddings is not None:
        return ("candle-layout checkpoints of an LM with depformer_low_rank_embeddings are not supported; load its safetensors "
                "checkpoint")
    return None


def normalize_lm_state_dict(sd: tp.Mapping[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    return _split_attention(_from_candle(sd))
