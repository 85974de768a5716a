"""Generates ``tests/golden/lm_tiny_cond.safetensors``: the 2B configuration's conditioning (``configs/moshi_dev_2b.json``: a LUT
conditioner on "description" fused by ``sum``), with and without classifier-free guidance, on the tiny LM through the
UNMODIFIED reference (CPU).  The conditioners run once per session outside the step (run_inference.py:38-56, lm.py:616-626);
what reaches the hot path is ``condition_sum`` [B or 2B, 1, dim], added to the summed input embeddings every step
(lm.py:398-399).  The fixture stores the reference's ``condition_sum`` and its tokens; the oracle restates the step.

    python -m oracle.gen_golden_cond          # build container only: needs $MOSHI_REFERENCE
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

COND_CFG = {"conditioners": {"description": {"type": "lut", "lut": {
    "n_bins": 31, "dim": 16, "tokenizer": "noop", "possible_values": ["very_bad", "bad", "neutral", "good", "very_good"]}}},
    "fuser": {"sum": ["description"]}}


@torch.no_grad()
def main() -> None:
    from moshi.conditioners import ConditionAttributes
    from moshi.models.lm import LMGen, LMModel
    from moshi.models.loaders import get_condition_fuser, get_conditioner_provider
    cfg = tiny_lm_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    torch.manual_seed(3)                                   # the conditioner's own (random-init) weights
    ref = LMModel(device="cpu", dtype=torch.bfloat16, condition_provider=get_conditioner_provider(cfg.dim, "cpu", COND_CFG),
                  fuser=get_condition_fuser(COND_CFG), **cfg.to_reference_kwargs()).eval()
    res = ref.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.startswith("condition_provider.") for k in res.missing_keys)
    B, steps = scenarios.CFG_B, scenarios.CFG_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps, seed=scenarios.CFG_SEED)
    # the conditioner's weights, under the checkpoint key names, so that moshi_b200.conditioners can be pinned on them
    cond_sd = {k: v.detach().clone() for k, v in ref.state_dict().items() if k.startswith("condition_provider.")}
    tensors, info = dict(cond_sd), {"generated_by": "oracle/gen_golden_cond.py", "torch": torch.__version__, "B": B, "steps": steps,
                         "none_marker": -3, "modes": {}}
    for name, cfg_coef in (("sum", 1.0), ("sum_cfg", 2.0)):
        conds = [ConditionAttributes(text={"description": "very_good"}, tensor={})] * B
        if cfg_coef != 1.0:                                # run_inference.py:44-50: the null half is "very_bad"
            conds = conds + [ConditionAttributes(text={"description": "very_bad"}, tensor={})] * B
        ct = ref.condition_provider.prepare_and_provide(conds)
        csum = ref.fuser.get_sum(ct).to(torch.bfloat16)
        gen = LMGen(ref, use_sampling=False, cfg_coef=cfg_coef, condition_tensors=ct)
        orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, cfg_coef=cfg_coef, condition_sum=csum)
        orc.streaming(B)
        outs, agree = [], True
        with gen.streaming(B):
            for i in range(steps):
                a, b = gen.step(codes[i]), orc.step(codes[i])
                assert (a is None) == (b is None), (name, i)
                outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if a is None else a)
                agree &= a is None or bool((a == b).all())
        tensors[name + ".tokens"] = torch.stack(outs)
        tensors[name + ".condition_sum"] = csum.contiguous()
        tensors[name + ".condition"] = ct["description"].condition.contiguous()          # fp32 [rows, 1, dim]
        tensors[name + ".mask"] = ct["description"].mask.to(torch.uint8).contiguous()
        info["modes"][name] = {"oracle_bit_exact_tokens": agree, "cfg_coef": cfg_coef}
    golden = ROOT / "tests" / "golden"
    save_file(tensors, golden / "lm_tiny_cond.safetensors")
    (golden / "lm_tiny_cond.json").write_text(json.dumps(info, indent=1))
    print(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
