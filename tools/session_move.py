#!/usr/bin/env python
"""Cost of moving one dialogue session between LM handles (``LMGen.export_session`` / ``import_session``) on the flagship 7B
geometry with synthetic weights, in one run:

* export of one session followed by its import into another handle, contiguous -> paged (pages of 64 slots) and
  paged -> contiguous, at fills 250 / 1500 / 3000, CUDA events over repeated calls after a warm-up;
* record bytes and achieved bandwidth: an export reads the session's rings and writes the record, an import reads the
  record and writes the rings, so a move moves 4 x the record bytes (against the H100 SXM data-sheet 3.35 TB/s);
* with two GPUs visible, the peer copy of the record to the second GPU (``record.to("cuda:1")``).

Prints the card's name and power limit, then one JSON object per measurement.  Needs an 80 GB H100 (two 7B handles).

    python tools/session_move.py
"""
from __future__ import annotations

import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

B, CTX, PAGE, ITERS, WARM = 2, 3000, 64, 10, 3
HBM_TBS = 3.35


def time_ms(fn, iters: int = ITERS, warm: int = WARM) -> float:
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    from moshi_b200.config import MOSHI_7B
    from moshi_b200.models import LMGen, loaders
    lms = [loaders.get_moshi_lm(None, MOSHI_7B.to_reference_kwargs(), device="cuda", synth_device="cuda") for _ in range(2)]
    contig, paged = LMGen(lms[0]), LMGen(lms[1])
    paged.kv_pool_frames, paged.kv_page_slots = B * -(-CTX // PAGE) * PAGE, PAGE
    contig.streaming_forever(B)
    paged.streaming_forever(B)
    peer = torch.cuda.device_count() > 1
    for fill in (250, 1500, 3000):
        contig.assume_fill(fill)
        paged.assume_fill(fill)
        for name, src, dst in (("contiguous->paged", contig, paged), ("paged->contiguous", paged, contig)):
            rec = src.export_session(0)
            n = rec.numel()
            export_ms = time_ms(lambda: src.export_session(0))
            import_ms = time_ms(lambda: dst.import_session(1, rec))
            move_ms = time_ms(lambda: dst.import_session(1, src.export_session(0)))
            line = {"what": "session_move", "direction": name, "fill": fill, "record_bytes": n,
                    "export_ms": round(export_ms, 3), "import_ms": round(import_ms, 3), "export_import_ms": round(move_ms, 3),
                    "move_gbs": round(4 * n / move_ms / 1e6, 1), "move_share_of_hbm": round(4 * n / move_ms / 1e9 / HBM_TBS, 3),
                    "export_gbs": round(2 * n / export_ms / 1e6, 1), "import_gbs": round(2 * n / import_ms / 1e6, 1)}
            if peer:
                line["peer_copy_ms"] = round(time_ms(lambda: rec.to("cuda:1")), 3)
            print(json.dumps(line), flush=True)
    if not peer:
        print(json.dumps({"what": "peer_copy", "measured": False, "reason": "one GPU visible"}), flush=True)


if __name__ == "__main__":
    main()
