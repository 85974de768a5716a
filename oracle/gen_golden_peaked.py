"""Generates ``tests/golden/lm_tiny_sampled_peaked.safetensors``: 30 sampled ``LMGen.step`` calls of the UNMODIFIED reference
(CPU, global Philox generator seeded with ``scenarios.LM_NOISE_SEED``) on the tiny LM with peaked output distributions
(``scenarios.peaked_state_dict``), with the exec-mask / reset events of ``scenarios.lm_mask_events``; records whether the oracle,
fed the same Exp(1) draws explicitly, reproduces every token.  Build container only (needs $MOSHI_REFERENCE):

    python -m oracle.gen_golden_peaked
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
from oracle import scenarios  # noqa: E402
from oracle.lm import LMOracle, LMSpec  # noqa: E402


@torch.no_grad()
def main() -> None:
    from moshi.models.lm import LMGen, LMModel
    cfg = tiny_lm_config()
    sd = scenarios.peaked_state_dict(cfg)
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **cfg.to_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.LM_B, scenarios.LM_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps)
    logits_rec, text_rec, audio_rec = [], [], []
    gen = LMGen(ref, use_sampling=True, temp=0.8, temp_text=0.7, on_text_logits_hook=lambda t: logits_rec.append(t.float().clone()),
                on_text_hook=lambda t: text_rec.append(t.clone()), on_audio_hook=lambda t: audio_rec.append(t.clone()))
    outs = []
    torch.manual_seed(scenarios.LM_NOISE_SEED)
    with gen.streaming(B):
        for i in range(steps):
            scenarios.lm_mask_events(gen, i, B)
            o = gen.step(codes[i])
            outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=True)
    orc.streaming(B)
    o_outs = []
    torch.manual_seed(scenarios.LM_NOISE_SEED)
    for i in range(steps):
        scenarios.lm_mask_events(orc, i, B)
        nt, na = scenarios.lm_noise(cfg, B)
        o = orc.step(codes[i], nt, na)
        o_outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
    tokens = torch.stack(outs)
    agree = bool((torch.stack(o_outs) == tokens).all())
    tl = torch.stack(logits_rec)[:, :, 0, 0]
    golden = ROOT / "tests" / "golden"
    # the raw decision of every sampler call (lm.py:736-757 hooks): text [steps, B], audio [steps, B, dep_q]
    save_file({"tokens": tokens, "text_logits": tl, "sampled_text": torch.stack(text_rec), "sampled_audio": torch.stack(audio_rec)},
              golden / "lm_tiny_sampled_peaked.safetensors")
    info = {"generated_by": "oracle/gen_golden_peaked.py", "torch": torch.__version__, "oracle_bit_exact_tokens": agree, "B": B,
            "steps": steps, "none_marker": -3, "peak_gain": scenarios.PEAK_GAIN, "text_logits_std": float(tl.std()),
            "distinct_text_tokens": int(tokens[:, :, 0].unique().numel())}
    (golden / "lm_tiny_sampled_peaked.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
