#!/usr/bin/env python
"""Cost of the paged temporal KV pool (``LMGen.kv_pool_frames``) on the flagship 7B configuration, in one run:

* ``attn_step_kernel`` (CUDA events), contiguous ring vs pages of 64 slots, 38 sessions x 32 heads, fills 750 / 1500 / 3000;
  the paged rows' pages interleave the way the step allocates them (page t of row b is the t-th page the pool handed out
  after t pages of every earlier row);
* the whole LM step, contiguous vs paged, 38 sessions at fill 3000 (every ring full), alternated twice;
* the LM step of 76 sessions in a pool the size of 38 full rings (the same KV bytes for twice the sessions).  A row at fill
  1500 holds 24 pages of 64 and 76 x 24 = 1824 exceeds the 38 x 47 = 1786 pages of 38 full rings, so those sessions run
  at fills 1440-1465 (23 pages each).

Prints the card's name and power limit, then one JSON object per measurement.  Needs an 80 GB H100.

    python tools/kv_pool.py
"""
from __future__ import annotations

import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from moshi_b200 import _lib  # noqa: E402

B, H, D, CTX, PAGE = 38, 32, 128, 3000, 64
FULL_RING = -(-CTX // PAGE) * PAGE          # slots of a full ring in whole pages (47 x 64)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def time_ms(fn, iters: int, warm: int = 5) -> float:
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


def attention(lib):
    T = -(-CTX // PAGE)
    qkv = torch.randn(B, 3 * H * D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, H, CTX, D, device="cuda").to(torch.bfloat16)
    v = torch.randn_like(k)
    kp = torch.randn(B * T, H, PAGE, D, device="cuda").to(torch.bfloat16)
    vp = torch.randn_like(kp)
    table = (torch.arange(T, dtype=torch.int32)[None, :] * B + torch.arange(B, dtype=torch.int32)[:, None]).cuda()
    out = torch.empty(B, H * D, device="cuda", dtype=torch.bfloat16)
    exec_ = torch.ones(B, dtype=torch.uint8, device="cuda")
    for fill in (750, 1500, 3000):
        pos = torch.full((B,), fill - 1, dtype=torch.int64, device="cuda")    # the step attends over `fill` keys
        res = {}
        for _ in range(2):                   # alternate, twice
            res.setdefault("contiguous", []).append(time_ms(lambda: _lib.check(lib.b200_op_attn_step(
                _lib.ptr(qkv), _lib.ptr(k), _lib.ptr(v), _lib.ptr(out), _lib.ptr(pos), _lib.ptr(exec_), B, H, CTX, 0, 10000.0,
                stream())), 200))
            res.setdefault("paged", []).append(time_ms(lambda: _lib.check(lib.b200_op_attn_step_paged(
                _lib.ptr(qkv), _lib.ptr(kp), _lib.ptr(vp), _lib.ptr(table), _lib.ptr(out), _lib.ptr(pos), _lib.ptr(exec_), B, H, CTX,
                PAGE, 0, 10000.0, stream())), 200))
        kv_bytes = 2 * B * H * fill * D * 2
        print(json.dumps({"what": "attn_step_kernel", "B": B, "H": H, "fill": fill, "page_slots": PAGE,
                          "contiguous_us": [round(t * 1e3, 2) for t in res["contiguous"]],
                          "paged_us": [round(t * 1e3, 2) for t in res["paged"]],
                          "kv_gbs_contiguous": round(kv_bytes / min(res["contiguous"]) / 1e6, 1),
                          "kv_gbs_paged": round(kv_bytes / min(res["paged"]) / 1e6, 1)}), flush=True)
    del k, v, kp, vp
    torch.cuda.empty_cache()


def lm_step_ms(lm, batch, fill, pool, steps=20):
    from moshi_b200.models import LMGen
    gen = LMGen(lm)
    gen.kv_pool_frames = pool
    g = torch.Generator().manual_seed(1)
    codes = [torch.randint(0, 2048, (batch, 8, 1), generator=g).cuda() for _ in range(4)]
    with gen.streaming(batch), torch.no_grad():
        gen.assume_fill(fill)
        for i in range(5):
            gen.step(codes[i % 4])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            gen.step(codes[i % 4])
        e1.record()
        torch.cuda.synchronize()
        flags = gen.error_flags()
        usage = gen.kv_pool_usage()
    assert not flags & 8, f"error flags {flags}"          # assume_fill's ungenerated token ring raises flag 1
    return e0.elapsed_time(e1) / steps, usage


def main():
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    lib = _lib.lib()
    attention(lib)

    from moshi_b200.config import MOSHI_7B
    from moshi_b200.models import loaders
    lm = loaders.get_moshi_lm(None, MOSHI_7B.to_reference_kwargs(), device="cuda", synth_device="cuda")
    torch.cuda.synchronize()
    res = {"contiguous": [], "paged": []}
    for _ in range(2):
        res["contiguous"].append(lm_step_ms(lm, B, CTX, None)[0])
        ms, usage = lm_step_ms(lm, B, CTX, B * FULL_RING)
        res["paged"].append(ms)
    print(json.dumps({"what": "lm_step", "B": B, "fill": CTX, "page_slots": PAGE, "pages": usage,
                      "contiguous_ms": [round(t, 3) for t in res["contiguous"]], "paged_ms": [round(t, 3) for t in res["paged"]],
                      "paged_over_contiguous": round(min(res["paged"]) / min(res["contiguous"]), 4)}), flush=True)
    ms, usage = lm_step_ms(lm, 2 * B, 1440, B * FULL_RING)
    print(json.dumps({"what": "lm_step_shared_pool", "B": 2 * B, "fill": "1440-1465", "pool_frames": B * FULL_RING, "page_slots": PAGE,
                      "pages": usage, "ms": round(ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
