"""Generates ``tests/golden/lm_tiny_sched.{json,safetensors}``: the depformer's weight-sharing schedule
(``depformer_weights_per_step_schedule``, lm.py:125-127, 172-181, transformer.py:291-316) and low-rank depformer embeddings
(``depformer_low_rank_embeddings``, lm.py:186-196, lm_utils.py:80-124) on the tiny LM (head dims 128 / 64), through the
UNMODIFIED reference (CPU).  A greedy and a sampled run, with the exec-mask and reset events of ``scenarios.lm_mask_events``;
the fixture records the reference's tokens and text logits and whether the oracle agrees bit for bit.

    MOSHI_REFERENCE=<checkout of kyutai-labs/moshi> python tools/gen_golden_sched.py
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
from oracle.lm import LMOracle  # noqa: E402
from tests.depformer_sched import sched_spec  # noqa: E402

SCHEDULE, RANK, SEED = [0, 1, 2, 2, 2, 3, 3, 3], 32, 57


def sched_config():
    return tiny_lm_config(depformer_weights_per_step_schedule=list(SCHEDULE), depformer_low_rank_embeddings=RANK)


@torch.no_grad()
def main() -> None:
    from moshi.models.lm import LMGen, LMModel
    cfg = sched_config()
    sd = synth_lm_state_dict(cfg, seed=SEED)
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **cfg.to_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.LM_B, scenarios.LM_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps, seed=SEED)
    tensors: dict[str, torch.Tensor] = {}
    info = {"generated_by": "tools/gen_golden_sched.py", "torch": torch.__version__, "B": B, "steps": steps, "seed": SEED,
            "noise_seed": scenarios.LM_NOISE_SEED, "schedule": SCHEDULE, "low_rank": RANK, "none_marker": -3, "runs": {}}
    for name, sampling in (("greedy", False), ("sampled", True)):
        logits: list[torch.Tensor] = []
        gen = LMGen(ref, use_sampling=sampling, temp=0.8, temp_text=0.7,
                    on_text_logits_hook=lambda t: logits.append(t[:, 0, 0].clone()))
        outs = []
        torch.manual_seed(scenarios.LM_NOISE_SEED)
        with gen.streaming(B):
            for i in range(steps):
                scenarios.lm_mask_events(gen, i, B)
                o = gen.step(codes[i])
                outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
        orc = LMOracle(sd, sched_spec(cfg), use_sampling=sampling)
        orc.streaming(B)
        o_outs, o_logits = [], []
        torch.manual_seed(scenarios.LM_NOISE_SEED)
        for i in range(steps):
            scenarios.lm_mask_events(orc, i, B)
            nt, na = scenarios.lm_noise(cfg, B) if sampling else (None, None)
            dbg: dict = {}
            o = orc.step(codes[i], nt, na, debug=dbg)
            o_logits.append(dbg["text_logits"][:, 0, 0])
            o_outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
        tokens, text_logits = torch.stack(outs), torch.stack(logits)
        tensors[f"{name}.tokens"] = tokens
        tensors[f"{name}.text_logits"] = text_logits.contiguous()
        info["runs"][name] = {"oracle_bit_exact_tokens": bool(torch.equal(torch.stack(o_outs), tokens)),
                              "oracle_bit_exact_text_logits": bool(torch.equal(torch.stack(o_logits), text_logits))}
    tensors["codes"] = codes
    golden = ROOT / "tests" / "golden"
    save_file(tensors, golden / "lm_tiny_sched.safetensors")
    (golden / "lm_tiny_sched.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
