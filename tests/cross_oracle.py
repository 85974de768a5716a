"""CPU restatement of cross-attention conditioning (test infrastructure), on top of ``oracle.lm.LMOracle``.

With ``cross_attention=True`` (the TTS models) every temporal layer runs, between its self-attention and its MLP
(``modules/transformer.py:779-798``), ``x = x + cross_attention(norm_cross(x), src, src)``:

* ``norm_cross`` is ``nn.LayerNorm(d, eps=1e-5)`` with weight and bias (``:727-732``);
* the query is ``x @ in_projs.0.weight[:d]^T``; keys and values are ``src @ in_projs.0.weight[d:]^T`` split as
  ``b t (p h d) -> p b h t d`` (``:495-505``), computed once per session and kept in ``_MHAState.k_cross / v_cross``
  (``:321-327, 518-531``);
* no RoPE, no mask, no causality: SDPA over all T keys (``:585``), then ``out_projs.0.weight``.

``src`` is ``fuser.get_cross(condition_tensors)`` in the model dtype (``models/lm.py:616-651``), one row per model row
(2B under classifier-free guidance).  ``_MHAState.reset`` does not clear the memory, and the TTS service replaces single rows
of it (``rust/moshi-server/tts.py:430-440``): ``set_condition_cross(src, rows)``.
"""
from __future__ import annotations

import typing as tp

import torch
import torch.nn.functional as F

from oracle import transformer as tr
from oracle.lm import LMOracle, scaled_embedding


def cross_kv(sd: dict, prefix: str, src: torch.Tensor, num_heads: int) -> tuple[torch.Tensor, torch.Tensor]:
    """``_compute_cross_attention`` (transformer.py:495-505): src [B, T, d] -> k, v [B, H, T, d / H]."""
    w = sd[prefix + ".cross_attention.in_projs.0.weight"]
    d = w.shape[1]
    kv = F.linear(src, w[d:])
    B, T, _ = kv.shape
    kv = kv.view(B, T, 2, num_heads, d // num_heads).permute(2, 0, 3, 1, 4)
    return kv[0], kv[1]


def cross_block(sd: dict, prefix: str, x: torch.Tensor, k: torch.Tensor, v: torch.Tensor, num_heads: int,
                taps: dict | None = None) -> torch.Tensor:
    """``_cross_attention_block`` (transformer.py:789-797) of one layer on x [B, S, d] against the cached k, v."""
    B, S, d = x.shape
    xn = F.layer_norm(x, (d,), sd[prefix + ".norm_cross.weight"], sd[prefix + ".norm_cross.bias"], 1e-5)
    w = sd[prefix + ".cross_attention.in_projs.0.weight"]
    q = F.linear(xn, w[:d]).view(B, S, num_heads, d // num_heads).transpose(1, 2)
    out = F.scaled_dot_product_attention(q, k, v, None, dropout_p=0.0)
    out = out.transpose(1, 2).reshape(B, S, d)
    if taps is not None:
        taps["norm_cross"], taps["cross_out"] = xn, out
    return x + F.linear(out, sd[prefix + ".cross_attention.out_projs.0.weight"])


class CrossLMOracle(LMOracle):
    """``LMOracle`` of an LM with cross-attention layers; ``condition_cross`` [MB, T, d] in the model dtype."""

    def __init__(self, sd: tp.Dict[str, torch.Tensor], spec, condition_cross: torch.Tensor, **kw):
        cfg_coef = kw.pop("cfg_coef", 1.0)
        super().__init__(sd, spec, **kw)
        self.cfg_coef = cfg_coef        # under CFG the condition's null half is in condition_cross (LMOracle only checks condition_sum)
        self.condition_cross = condition_cross
        self.layer_taps: list[dict] | None = None

    def streaming(self, batch: int) -> None:
        super().streaming(batch)
        assert self.condition_cross.shape[0] == self.model_batch, "cfg requires 2x more conditions."    # lm.py:650-651
        self.memory = [cross_kv(self.sd, f"transformer.layers.{i}", self.condition_cross, self.spec.num_heads)
                       for i in range(self.spec.num_layers)]

    def set_condition_cross(self, src: torch.Tensor, rows: tp.Sequence[int]) -> None:
        """tts.py:430-440: every layer's ``k_cross[rows] = k`` / ``v_cross[rows] = v`` of the new source."""
        idx = torch.tensor(list(rows), dtype=torch.long)
        for i, (k, v) in enumerate(self.memory):
            nk, nv = cross_kv(self.sd, f"transformer.layers.{i}", src, self.spec.num_heads)
            k.index_copy_(0, idx, nk)
            v.index_copy_(0, idx, nv)

    def forward_text(self, tokens: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """``LMOracle.forward_text`` with the temporal transformer's layers restated (``tr.forward``) plus the cross block.
        With ``layer_taps`` set to a list, each layer appends its activations (the GPU handle's taps)."""
        s = self.spec
        x = None
        for k in range(s.n_q):
            e = scaled_embedding(self.sd, f"emb.{k}", tokens[:, k + 1])
            x = e if x is None else x + e
        t = scaled_embedding(self.sd, "text_emb", tokens[:, 0])
        x = t if x is None else x + t
        if self.condition_sum is not None:
            x = x + self.condition_sum.to(x)
        spec, st = self.main_spec, self.main_state
        assert spec.positional_embedding == "rope" and not spec.layer_scale and not spec.weights_per_step
        T = x.shape[1]
        for li, ls in enumerate(st.layers):
            p = f"transformer.layers.{li}"
            taps = {} if self.layer_taps is not None else None
            upd = tr.attention(self.sd, p + ".self_attn", spec, tr.apply_norm(spec.norm, x, self.sd, p + ".norm1"), ls, st)
            x = x.to(upd) + upd
            if taps is not None:
                taps["x_attn"] = x
            x = cross_block(self.sd, p, x, self.memory[li][0], self.memory[li][1], s.num_heads, taps)
            if taps is not None:
                taps["x_cross"] = x
            upd = tr.feed_forward(self.sd, p, spec, tr.apply_norm(spec.norm, x, self.sd, p + ".norm2"), ls.offset_cpu)
            x = x.to(upd) + upd
            if taps is not None:
                taps["x_out"] = x
                self.layer_taps.append(taps)
            ls.offset_cpu += T
        st.offsets[:] = torch.where(st.exec_mask, st.offsets + T, st.offsets)
        out = tr.apply_norm(s.norm, x, self.sd, "out_norm")
        logits = F.linear(out, self.sd["text_linear.weight"], self.sd.get("text_linear.bias"))
        return out, logits[:, None]
