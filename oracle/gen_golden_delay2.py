"""Generates ``tests/golden/lm_tiny_delay2.safetensors``: a member of the family with the acoustic delay pattern of the 2B
configuration (``configs/moshi_dev_2b.json``: delays up to 2) run through the UNMODIFIED reference (CPU), and records whether
the oracle agrees bit for bit.  Build container only (needs $MOSHI_REFERENCE):

    python -m oracle.gen_golden_delay2
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

os.environ["NO_TORCH_COMPILE"] = "1"
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, os.path.join(os.environ.get("MOSHI_REFERENCE", ""), "moshi"))   # a checkout of kyutai-labs/moshi

import torch  # noqa: E402
from safetensors.torch import save_file  # noqa: E402

from moshi_b200.synth import synth_lm_state_dict  # noqa: E402
from oracle import scenarios  # noqa: E402
from oracle.lm import LMOracle, LMSpec  # noqa: E402


@torch.no_grad()
def main() -> None:
    from moshi.models.lm import LMGen, LMModel
    cfg = scenarios.delay2_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.DELAY2_SEED)
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **cfg.to_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.DELAY2_B, scenarios.DELAY2_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps, seed=scenarios.DELAY2_SEED)
    gen = LMGen(ref, use_sampling=False)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False)
    orc.streaming(B)
    outs, agree = [], True
    with gen.streaming(B):
        for i in range(steps):
            a, b = gen.step(codes[i]), orc.step(codes[i])
            assert (a is None) == (b is None), i
            outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if a is None else a)
            agree &= a is None or bool((a == b).all())
    golden = ROOT / "tests" / "golden"
    save_file({"tokens": torch.stack(outs)}, golden / "lm_tiny_delay2.safetensors")
    info = {"generated_by": "oracle/gen_golden_delay2.py", "torch": torch.__version__, "oracle_bit_exact_tokens": agree, "B": B,
            "steps": steps, "none_marker": -3, "delays": list(cfg.delays)}
    (golden / "lm_tiny_delay2.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
