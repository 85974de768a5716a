"""Generates ``tests/golden/lm_tiny_cfg.safetensors``: classifier-free guidance without a conditioner (``LMGen(cfg_coef != 1,
cfg_is_no_text / cfg_is_masked_until)``, lm.py:596-604, 646-662, 714-732, 820-833) on the tiny LM, run through the UNMODIFIED
reference (CPU); records whether the oracle agrees bit for bit.  Build container only (needs $MOSHI_REFERENCE):

    python -m oracle.gen_golden_cfg

Oracle groundwork for SURVEY.md 8(f) item 2; the CUDA path does not build CFG yet.
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

from moshi_b200.config import tiny_lm_config  # noqa: E402
from moshi_b200.synth import synth_lm_state_dict  # noqa: E402
from oracle import scenarios  # noqa: E402
from oracle.lm import LMOracle, LMSpec  # noqa: E402


@torch.no_grad()
def main() -> None:
    from moshi.models.lm import LMGen, LMModel
    cfg = tiny_lm_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **cfg.to_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.CFG_B, scenarios.CFG_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps, seed=scenarios.CFG_SEED)
    tensors, info = {}, {"generated_by": "oracle/gen_golden_cfg.py", "torch": torch.__version__, "B": B, "steps": steps,
                         "none_marker": -3, "modes": {}}
    for name, kw in scenarios.CFG_MODES.items():
        gen = LMGen(ref, use_sampling=False, **kw)
        orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, **kw)
        orc.streaming(B)
        outs, agree = [], True
        with gen.streaming(B):
            for i in range(steps):
                if i == scenarios.CFG_RESET_STEP:
                    r = torch.tensor([True, False])
                    gen.reset_streaming(r)
                    orc.reset_streaming(r)
                a, b = gen.step(codes[i]), orc.step(codes[i])
                assert (a is None) == (b is None), (name, i)
                outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if a is None else a)
                agree &= a is None or bool((a == b).all())
        tensors[name] = torch.stack(outs)
        info["modes"][name] = {"oracle_bit_exact_tokens": agree, **{k: v for k, v in kw.items()}}
    golden = ROOT / "tests" / "golden"
    save_file(tensors, golden / "lm_tiny_cfg.safetensors")
    (golden / "lm_tiny_cfg.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
