"""Generates ``tests/golden/lm_tiny_cross.{json,safetensors}``: cross-attention conditioning (the TTS models' LM:
``cross_attention=True``, a tensor conditioner fused by ``cross``) on the tiny LM through the UNMODIFIED reference (CPU).

Two fuser modes, without and with ``cross_attention_pos_emb``; in each, a greedy run, a sampled run and a classifier-free
guidance run (the null half: nulled attributes, i.e. learnt padding everywhere).  Row 1's condition is shorter than the
others (masked positions: learnt padding).  At ``reset_step`` row 1 takes a new condition the way the TTS service does it
(``rust/moshi-server/tts.py:430-440``: ``k_cross[rows] = k``, ``v_cross[rows] = v`` of every cross-attention module) and is
reset.  The runs are longer than the context, so the temporal rings wrap.

The fixture stores the reference's ``condition_cross``, the replacement source, the conditioner inputs and weights, its
tokens and its text logits; ``tests/cross_oracle.py`` restates the step.

    MOSHI_REFERENCE=<checkout of kyutai-labs/moshi> python tools/gen_golden_cross.py
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

os.environ["NO_TORCH_COMPILE"] = "1"
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, os.path.join(os.environ.get("MOSHI_REFERENCE", ""), "moshi"))

import torch  # noqa: E402
from safetensors.torch import save_file  # noqa: E402

from moshi_b200.config import tiny_lm_config  # noqa: E402
from moshi_b200.synth import synth_lm_state_dict  # noqa: E402
from oracle import scenarios  # noqa: E402
from oracle.lm import LMSpec  # noqa: E402
from tests.cross_oracle import CrossLMOracle  # noqa: E402

B, STEPS, RESET_STEP, SWAP_ROW = 3, 16, 6, 1
COND_DIM, T_FULL, T_SHORT = 64, 10, 7
SEED, NOISE_SEED = 31, 77
FUSERS = {
    "cross": {"cross": ["speaker_wavs"]},
    "cross_pos": {"cross": ["speaker_wavs"], "cross_attention_pos_emb": True, "cross_attention_pos_emb_scale": 0.5},
}
RUNS = {"greedy": dict(use_sampling=False, cfg_coef=1.0), "sampled": dict(use_sampling=True, cfg_coef=1.0),
        "cfg": dict(use_sampling=False, cfg_coef=2.0)}


def lm_config(fuser: dict):
    return tiny_lm_config(cross_attention=True, fuser=fuser,
                          conditioners={"speaker_wavs": {"type": "tensor", "tensor": {"dim": COND_DIM}}})


def voices() -> tuple[list[torch.Tensor], torch.Tensor]:
    """One speaker tensor [1, T, COND_DIM] per session (row 1 shorter) and the one row SWAP_ROW takes at RESET_STEP."""
    g = torch.Generator().manual_seed(SEED)
    v = [torch.randn(1, T_SHORT if b == SWAP_ROW else T_FULL, COND_DIM, generator=g) for b in range(B)]
    return v, torch.randn(1, T_FULL, COND_DIM, generator=g)


@torch.no_grad()
def main() -> None:
    from moshi.conditioners import ConditionAttributes, TensorCondition
    from moshi.models.lm import LMGen, LMModel
    from moshi.models.loaders import get_condition_fuser, get_conditioner_provider

    def attrs(t: torch.Tensor, null: bool = False):
        cond = TensorCondition(torch.zeros_like(t), torch.zeros(1, t.shape[1], dtype=torch.bool)) if null \
            else TensorCondition.from_tensor(t)
        return ConditionAttributes(text={}, tensor={"speaker_wavs": cond})

    vs, swap = voices()
    tensors: dict[str, torch.Tensor] = {}
    info = {"generated_by": "tools/gen_golden_cross.py", "torch": torch.__version__, "B": B, "steps": STEPS,
            "reset_step": RESET_STEP, "swap_row": SWAP_ROW, "cond_dim": COND_DIM, "noise_seed": NOISE_SEED, "none_marker": -3,
            "fusers": FUSERS, "runs": RUNS, "modes": {}}
    for b, v in enumerate(vs):
        tensors[f"voice.{b}"] = v.contiguous()
    tensors["voice.swap"] = swap.contiguous()
    for fname, fuser in FUSERS.items():
        cfg = lm_config(fuser)
        sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
        full = {"conditioners": cfg.conditioners, "fuser": cfg.fuser}
        ref = LMModel(device="cpu", dtype=torch.bfloat16, condition_provider=get_conditioner_provider(cfg.dim, "cpu", full),
                      fuser=get_condition_fuser(full), **cfg.to_reference_kwargs()).eval()
        ref.load_state_dict(sd, strict=True)
        for k, v in ref.state_dict().items():
            if k.startswith("condition_provider."):
                tensors[f"{fname}.{k}"] = v.detach().clone().contiguous()
        codes = scenarios.lm_input_codes(cfg, B, STEPS, seed=SEED)
        tensors[f"{fname}.codes"] = codes
        cross_modules = [layer.cross_attention for layer in ref.transformer.layers]
        for rname, run in RUNS.items():
            cfg_on = run["cfg_coef"] != 1.0
            conds = [attrs(v) for v in vs] + ([attrs(v, null=True) for v in vs] if cfg_on else [])
            ct = ref.condition_provider.prepare_and_provide(conds)
            cross = ref.fuser.get_cross(ct).to(torch.bfloat16)
            swap_src = ref.fuser.get_cross(ref.condition_provider.prepare_and_provide([attrs(swap)])).to(torch.bfloat16)
            logits: list[torch.Tensor] = []
            gen = LMGen(ref, use_sampling=run["use_sampling"], cfg_coef=run["cfg_coef"], condition_tensors=ct,
                        on_text_logits_hook=lambda t: logits.append(t[:, 0, 0].clone()))
            orc = CrossLMOracle(sd, LMSpec.from_config(cfg), condition_cross=cross.clone(), use_sampling=run["use_sampling"],
                                cfg_coef=run["cfg_coef"])
            runs = {}
            for who in ("ref", "oracle"):
                torch.manual_seed(NOISE_SEED)
                outs, logs = [], []
                ctx = gen.streaming(B) if who == "ref" else None
                if ctx is None:
                    orc.streaming(B)
                else:
                    ctx.__enter__()
                logits.clear()
                for i in range(STEPS):
                    if i == RESET_STEP:                         # tts.py:430-440, then the row's reset
                        mask = torch.zeros(B, dtype=torch.bool)
                        mask[SWAP_ROW] = True
                        if who == "ref":
                            for m in cross_modules:
                                k, v = m._compute_cross_attention(swap_src, swap_src)
                                m._streaming_state.k_cross.index_copy_(0, torch.tensor([SWAP_ROW]), k)
                                m._streaming_state.v_cross.index_copy_(0, torch.tensor([SWAP_ROW]), v)
                            gen.reset_streaming(mask)
                        else:
                            orc.set_condition_cross(swap_src, [SWAP_ROW])
                            orc.reset_streaming(mask)
                    if who == "ref":
                        out = gen.step(codes[i])
                    else:
                        dbg: dict = {}
                        out = orc.step(codes[i], debug=dbg)
                        logs.append(dbg["text_logits"][:, 0, 0])
                    outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if out is None else out)
                if ctx is not None:
                    ctx.__exit__(None, None, None)
                runs[who] = (torch.stack(outs), torch.stack(logits if who == "ref" else logs))
            name = f"{fname}.{rname}"
            tensors[name + ".tokens"] = runs["ref"][0]
            tensors[name + ".text_logits"] = runs["ref"][1].contiguous()
            tensors[name + ".condition_cross"] = cross.contiguous()
            tensors[name + ".swap_cross"] = swap_src.contiguous()
            tensors[name + ".condition"] = ct["speaker_wavs"].condition.contiguous()
            tensors[name + ".mask"] = ct["speaker_wavs"].mask.to(torch.uint8).contiguous()
            info["modes"][name] = {"oracle_bit_exact_tokens": bool(torch.equal(runs["ref"][0], runs["oracle"][0])),
                                   "oracle_bit_exact_text_logits": bool(torch.equal(runs["ref"][1], runs["oracle"][1]))}
    golden = ROOT / "tests" / "golden"
    save_file(tensors, golden / "lm_tiny_cross.safetensors")
    (golden / "lm_tiny_cross.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info["modes"], indent=1))


if __name__ == "__main__":
    main()
