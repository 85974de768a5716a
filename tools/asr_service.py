#!/usr/bin/env python
"""Batched speech-to-text service (``serving.ASRService``) at serving batch: ms per 80 ms frame and the slots one GPU sustains.

    python tools/asr_service.py [--batches 32,64,128,256] [--frames 60] [--warmup 10] [--fill 375]

Every slot is ACTIVE with random PCM, Mimi encodes 32 codebooks, and the LM is STT-shaped with synthetic weights.  The
reference's STT configs (configs/stt_*.json) carry no model dimensions, so the geometry below is ASSUMED and printed with the
results.  The LM's rings are declared full (``--fill``, the steady state of a stream longer than context / 12.5 s).

Per batch size it reports the wall clock of ``step`` (host clock around a call that ends in its own host wait; p50 / p90 over
``--frames`` frames after ``--warmup``), and a split of the frame: Mimi's encode and the LM step timed on their own with CUDA
events at the same batch (medians), the rest (H2D / D2H, masks, flags, host work) being the wall-clock p50 minus both.  A slot
count is sustained when the p90 frame fits in 80 ms.  Prints the card's name and power limit, then one JSON object per batch.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

ASSUMED = dict(dim=2048, num_layers=16, num_heads=16, n_q=32, dep_q=0, card=2048, text_card=8000, context=375,
               hidden_scale=4.125, delays=[0] * 33, extra_heads_num_heads=4, extra_heads_dim=6)
FRAME_MS = 80.0


def _events_ms(fn, n):
    times = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def measure(B, lm, mimi, frames, warmup, fill):
    from moshi_b200.serving import ACTIVE, ASRService
    svc = ASRService(B, lm, mimi, asr_delay_in_tokens=32)
    svc.lm_gen.assume_fill(fill)
    g = np.random.default_rng(B)
    pcm = [(0.1 * g.standard_normal(B * mimi.frame_size)).astype(np.float32) for _ in range(8)]
    flags, toks = np.zeros(B, np.uint8), np.zeros(B, np.uint32)
    heads = np.zeros((B, lm.cfg.extra_heads_num_heads), np.float32)
    upd = [ACTIVE] * B
    wall = []
    for i in range(warmup + frames):
        t0 = time.perf_counter()
        svc.step(pcm[i % len(pcm)], flags, toks, heads, upd)
        if i >= warmup:
            wall.append((time.perf_counter() - t0) * 1e3)
    # the two device stages on their own, same handles, same batch
    x = torch.from_numpy(pcm[0]).cuda().view(B, 1, mimi.frame_size)
    codes = mimi.encode(x)
    for _ in range(warmup):
        svc.lm_gen.step_with_extra_heads(codes)
    enc = _events_ms(lambda: mimi.encode(x), frames)
    step = _events_ms(lambda: svc.lm_gen.step_with_extra_heads(codes), frames)
    svc.close()
    p50, p90 = float(np.percentile(wall, 50)), float(np.percentile(wall, 90))
    return dict(slots=B, frame_ms_p50=round(p50, 3), frame_ms_p90=round(p90, 3), encode_ms=round(enc, 3), lm_step_ms=round(step, 3),
                rest_ms=round(p50 - enc - step, 3), within_80ms=p90 <= FRAME_MS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,64,128,256")
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--fill", type=int, default=ASSUMED["context"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tools/asr_service.py measures on a GPU; none is visible")
    from moshi_b200.config import MimiConfig, tiny_lm_config
    from moshi_b200.models import LMModel, MimiModel
    from moshi_b200.synth import iter_synth_lm_tensors, synth_mimi_state_dict
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    print(json.dumps({"assumed_lm_geometry": ASSUMED, "mimi_codebooks": 32, "weights": "synthetic"}), flush=True)
    cfg = tiny_lm_config(**ASSUMED)
    lm = LMModel(cfg, iter_synth_lm_tensors(cfg, seed=1, device="cuda"), device="cuda")
    mcfg = MimiConfig(num_codebooks=32)
    mimi = MimiModel(mcfg, synth_mimi_state_dict(mcfg, seed=1234), device="cuda")
    rows = []
    for B in (int(b) for b in args.batches.split(",")):
        r = measure(B, lm, mimi, args.frames, args.warmup, args.fill)
        rows.append(r)
        print(json.dumps(r), flush=True)
    ok = [r["slots"] for r in rows if r["within_80ms"]]
    print(json.dumps({"slots_sustained_within_80ms": max(ok) if ok else 0, "of_measured": [r["slots"] for r in rows]}), flush=True)
    print(f"\n{'slots':>6} {'p50 ms':>8} {'p90 ms':>8} {'encode':>8} {'LM step':>8} {'rest':>8}  within 80 ms")
    for r in rows:
        print(f"{r['slots']:>6} {r['frame_ms_p50']:>8.2f} {r['frame_ms_p90']:>8.2f} {r['encode_ms']:>8.2f} {r['lm_step_ms']:>8.2f} "
              f"{r['rest_ms']:>8.2f}  {'yes' if r['within_80ms'] else 'no'}")


if __name__ == "__main__":
    main()
