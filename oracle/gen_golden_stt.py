"""Generates ``tests/golden/lm_stt_tiny.safetensors`` by running the UNMODIFIED reference (CPU) on the STT-style scenario of
``oracle/scenarios.py`` (no depformer, ``extra_heads``; ``LMGen.step_with_extra_heads``, lm.py:793-807 — what
``rust/moshi-server/batched_asr.py:197`` calls), and records whether the oracle agrees bit for bit.

    python -m oracle.gen_golden_stt          # build container only: needs $MOSHI_REFERENCE

Test infrastructure for the next row of SURVEY.md 8(f) item 2; the CUDA path does not implement this configuration yet.
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

from oracle import scenarios  # noqa: E402
from oracle.lm import LMOracle  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"


@torch.no_grad()
def main() -> None:
    from moshi.models.lm import LMGen, LMModel
    sd = scenarios.stt_state_dict()
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **scenarios.stt_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.STT_B, scenarios.STT_STEPS
    codes = scenarios.stt_input_codes()
    gen = LMGen(ref, use_sampling=False, temp=0.0, temp_text=0.0)
    orc = LMOracle(sd, scenarios.stt_spec(), use_sampling=False)
    orc.streaming(B)
    toks, heads, agree = [], [], True
    with gen.streaming(B):
        for i in range(steps):
            if i == 6:                                   # slot 1 is recycled, like ASRService.step's RESET (batched_asr.py:154-158)
                r = torch.tensor([False, True])
                gen.reset_streaming(r)
                orc.reset_streaming(r)
            got = gen.step_with_extra_heads(codes[i])
            want = orc.step_with_extra_heads(codes[i])
            assert (got is None) == (want is None), i
            if got is None:
                toks.append(torch.full((B, 1, 1), -3, dtype=torch.long))
                heads.append(torch.zeros(2, B, 6))
                continue
            t, hs = got
            toks.append(t)
            heads.append(torch.stack([h[:, 0].float() for h in hs]))
            agree &= bool((t == want[0]).all()) and all(torch.equal(a, b) for a, b in zip(hs, want[1]))
    save_file({"tokens": torch.stack(toks), "extra_heads": torch.stack(heads)}, GOLDEN / "lm_stt_tiny.safetensors")
    info = {"generated_by": "oracle/gen_golden_stt.py", "torch": torch.__version__, "oracle_bit_exact": agree, "B": B,
            "steps": steps, "none_marker": -3}
    (GOLDEN / "lm_stt_tiny.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
