"""Generates ``tests/golden/*`` by running the UNMODIFIED reference (``$MOSHI_REFERENCE/moshi``, CPU).

Run in the build container only (needs a checkout of the reference, ``MOSHI_REFERENCE``):

    python -m oracle.gen_golden

For every scenario the script (1) runs the reference, (2) runs the oracle on the same synthetic
weights and inputs and records whether they agree bit for bit, (3) stores the reference outputs as
small safetensors fixtures.  ``tests/golden/MANIFEST.json`` records torch version, seeds and the
agreement flags; the ``-m "not gpu"`` tests re-check the oracle against the fixtures, the ``-m gpu``
tests check the CUDA path against the same fixtures.
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

from moshi_b200.config import MimiConfig, tiny_lm_config  # noqa: E402
from moshi_b200.synth import synth_lm_state_dict, synth_mimi_state_dict  # noqa: E402
from oracle.lm import LMOracle, LMSpec  # noqa: E402
from oracle.mimi import MimiOracle  # noqa: E402
from oracle import scenarios  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"


@torch.no_grad()
def mimi_fixtures(manifest: dict) -> None:
    from moshi.models import loaders
    cfg = MimiConfig()
    sd = synth_mimi_state_dict(cfg, seed=scenarios.MIMI_SEED)
    ref = loaders.get_mimi(None, device="cpu", num_codebooks=cfg.num_codebooks)
    ref.load_state_dict(sd, strict=True)

    # --- config 1: 1 s 440 Hz sine, B=1 (BASELINE.json configs[0]) -------------------------
    sine = scenarios.sine_1s()
    codes_batch = ref.encode(scenarios.sine_1s_full())   # non-streaming, 24000 samples: pads to 13 frames
    pcm_batch = ref.decode(codes_batch)
    n = sine.shape[-1] // cfg.frame_size
    cs, ps = [], []
    with ref.streaming(1):
        for f in range(n):
            c = ref.encode(sine[..., f * 1920:(f + 1) * 1920])
            cs.append(c)
            ps.append(ref.decode(c))
    codes_stream, pcm_stream = torch.cat(cs, -1), torch.cat(ps, -1)
    orc = MimiOracle(sd, cfg)
    orc.streaming(1)
    oc, op = [], []
    for f in range(n):
        c = orc.encode(sine[..., f * 1920:(f + 1) * 1920])
        oc.append(c)
        op.append(orc.decode(c))
    agree = bool((torch.cat(oc, -1) == codes_stream).all()) and bool((torch.cat(op, -1) == pcm_stream).all())
    save_file({"codes_batch": codes_batch, "pcm_batch": pcm_batch, "codes_stream": codes_stream,
               "pcm_stream": pcm_stream}, GOLDEN / "mimi_sine.safetensors")
    manifest["mimi_sine"] = {
        "oracle_bit_exact": agree, "frames": n,
        "distinct_codes": int(codes_stream.unique().numel()),
        "stream_vs_batch_codes_equal": bool((codes_stream == codes_batch[..., :n]).all()),
        "stream_vs_batch_pcm_maxabs": float((pcm_stream - pcm_batch[..., :pcm_stream.shape[-1]]).abs().max()),
    }

    # --- masked / reset scenario, B=3 (scripts/test_missing_data.py pattern) --------------------
    B, frames = scenarios.MIMI_MASK_B, scenarios.MIMI_MASK_FRAMES
    pcm = scenarios.mimi_noise(B, frames)
    cs, ps, lat = [], [], []
    with ref.streaming(B):
        for f in range(frames):
            scenarios.mimi_mask_events(ref, f, B)
            x = pcm[..., f * 1920:(f + 1) * 1920]
            c = ref.encode(x)
            cs.append(c)
            ps.append(ref.decode(c))
    orc = MimiOracle(sd, cfg)
    orc.streaming(B)
    oc, op = [], []
    for f in range(frames):
        scenarios.mimi_mask_events(orc, f, B)
        c = orc.encode(pcm[..., f * 1920:(f + 1) * 1920])
        oc.append(c)
        op.append(orc.decode(c))
    codes, out = torch.stack(cs), torch.stack(ps)
    agree = bool((torch.stack(oc) == codes).all()) and bool((torch.stack(op) == out).all())
    save_file({"codes": codes, "pcm": out}, GOLDEN / "mimi_masked.safetensors")
    manifest["mimi_masked"] = {"oracle_bit_exact": agree, "B": B, "frames": frames,
                               "distinct_codes": int(codes.unique().numel())}


@torch.no_grad()
def lm_fixtures(manifest: dict) -> None:
    from moshi.models.lm import LMGen, LMModel
    cfg = tiny_lm_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    ref = LMModel(device="cpu", dtype=torch.bfloat16, **cfg.to_reference_kwargs()).eval()
    ref.load_state_dict(sd, strict=True)
    B, steps = scenarios.LM_B, scenarios.LM_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps)

    for name, use_sampling in (("lm_tiny_sampled", True), ("lm_tiny_greedy", False)):
        logits_rec = []
        gen = LMGen(ref, use_sampling=use_sampling, temp=0.8, temp_text=0.7,
                    on_text_logits_hook=lambda t: logits_rec.append(t.float().clone()))
        outs = []
        torch.manual_seed(scenarios.LM_NOISE_SEED)
        with gen.streaming(B):
            for i in range(steps):
                scenarios.lm_mask_events(gen, i, B)
                o = gen.step(codes[i])
                outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
        orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=use_sampling)
        orc.streaming(B)
        o_outs = []
        torch.manual_seed(scenarios.LM_NOISE_SEED)
        for i in range(steps):
            scenarios.lm_mask_events(orc, i, B)
            nt, na = scenarios.lm_noise(cfg, B) if use_sampling else (None, None)
            o = orc.step(codes[i], nt, na)
            o_outs.append(torch.full((B, cfg.dep_q + 1, 1), -3, dtype=torch.long) if o is None else o)
        tokens = torch.stack(outs)
        agree = bool((torch.stack(o_outs) == tokens).all())
        save_file({"tokens": tokens, "text_logits": torch.stack(logits_rec)[:, :, 0, 0]},
                  GOLDEN / f"{name}.safetensors")
        manifest[name] = {"oracle_bit_exact_tokens": agree, "B": B, "steps": steps,
                          "none_marker": -3}


def main() -> None:
    GOLDEN.mkdir(parents=True, exist_ok=True)
    manifest: dict = {
        "generated_by": "oracle/gen_golden.py", "torch": torch.__version__,
        "reference": "kyutai-labs/moshi python package (moshi 0.2.x, unmodified, CPU, NO_TORCH_COMPILE=1)",
        "reference_test_lm": "copied verbatim from the reference's moshi/tests/assets (KAT of tests/test_lm.py)",
    }
    mimi_fixtures(manifest)
    lm_fixtures(manifest)
    with open(GOLDEN / "MANIFEST.json", "w") as f:
        json.dump(manifest, f, indent=1)
    print(json.dumps(manifest, indent=1))


if __name__ == "__main__":
    main()
