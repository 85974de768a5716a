"""Cost of per-session sampling on the Moshi 7B LM step (synthetic weights), timed with CUDA events after warm-up.

At 1 and 38 sessions on full 3000-slot rings (assume_fill) and at 128 sessions on rings shortened to fit (kv_capacity), three
cases: off (a plain handle); on with every row at the handle-wide values; on with every row at
repetition penalty 1.2, context 200 and a pad bias.  Also the text path alone: the device time per step of
text_adjust_kernel, sample_text_kernel and every sample_kernel launch (the launch chain's audio samplers are sample_kernel
too), from a separate profiled run.  "off" is a plain handle; the two "on" cases share one session-sampling handle and
alternate window by window on the same rings.  The two handles run one after the other, each on its own rings (two sets of
full rings do not fit at once), so off-versus-on step times carry the machine's drift between them and the text-path column
is the direct cost.  Prints the card's name and power limit first.

    python tools/session_sampling.py [--steps 30] [--warmup 5] [--sessions 1,38,128]
"""
from __future__ import annotations

import argparse
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402


def card_info() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return q or torch.cuda.get_device_name()


def ev_time(fn, iters: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3      # us


def main() -> None:
    from moshi_b200.config import MOSHI_7B
    from moshi_b200.models import LMGen, loaders
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sessions", default="1,38,128")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card_info()}", flush=True)
    lm = loaders.get_moshi_lm(None, MOSHI_7B.to_reference_kwargs(), device=dev, synth_device=dev)
    ctx = MOSHI_7B.context
    rows = []
    for B in [int(x) for x in args.sessions.split(",")]:
        free = torch.cuda.mem_get_info(dev)[0]
        per_slot = 32 * 2 * 4096 * 2                             # K and V of 32 layers, bf16, one model row
        room = free - 2.5e9                                      # activations, workspaces and streaming_begin's 1 GiB margin
        cap = ctx if B * ctx * per_slot < room else int(room // (B * per_slot))
        fill = min(ctx, cap)
        cases = ("off", "on, defaults", "on, penalised")
        times = {k: [] for k in cases}
        text = {}
        codes = torch.randint(0, 2048, (B, 8, 1), device=dev)

        def settle(g, name):                                      # the case's settings on every row of the "on" handle
            if name == "on, penalised":
                g.set_session_sampling(range(B), pad_mult=1.0, repetition_context=200, repetition_penalty=1.2)
            elif name == "on, defaults":
                g.set_session_sampling(range(B))

        # two handles, one streaming at a time (each holds its own full rings): "off", then "on", whose two cases alternate
        # round by round on the same rings
        for handle, names in (("off", cases[:1]), ("on", cases[1:])):
            g = LMGen(lm, use_sampling=True)
            g.kv_capacity = None if cap >= ctx else cap
            g.session_sampling = 200 if handle == "on" else None
            g.streaming_forever(B)
            g.assume_fill(fill - len(names) * (args.warmup + args.rounds * args.steps + 5) - 2)     # a short ring never overflows
            for name in names:
                settle(g, name)
                for _ in range(args.warmup):
                    g.step(codes)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for name in names:
                    settle(g, name)
                    times[name].append(ev_time(lambda: g.step(codes), args.steps))
            for name in names:                                    # the text path alone: its kernels' device time per step
                settle(g, name)
                n_prof = 5
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(n_prof):
                        g.step(codes)
                    torch.cuda.synchronize()
                us = 0.0
                for e in prof.key_averages():
                    if any(k in e.key for k in ("text_adjust_kernel", "sample_text_kernel", "sample_kernel")):
                        us += e.device_time_total / n_prof
                text[name] = us
            g._stop()
        for name in cases:
            t = np.array(times[name]) / 1e3
            rows.append((B, fill, name, t.mean(), t.min(), t.max(), text[name]))
            print(f"B={B:4d} fill={fill:5d} {name:14s} step {t.mean():8.3f} ms (min {t.min():.3f}, max {t.max():.3f})  "
                  f"text path {text[name]:8.1f} us", flush=True)
    print("\n| sessions | ring fill | case | step ms (mean of rounds) | min | max | text path us |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r[0]} | {r[1]} | {r[2]} | {r[3]:.3f} | {r[4]:.3f} | {r[5]:.3f} | {r[6]:.1f} |")


if __name__ == "__main__":
    main()
