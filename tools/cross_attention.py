#!/usr/bin/env python
"""Cost of cross-attention conditioning (``cross_attention=True``, the TTS models' LM) on an ASSUMED TTS-like geometry with
synthetic weights: dim 2048, 16 heads (D = 128), 16 temporal layers, context 500, n_q = 32, dep_q = 16, condition memories of
T = 125 and 625 keys, at 32 / 64 / 128 / 256 sessions.  The geometry is not read from a released checkpoint; only its
shape matters for timing.  In one run:

* the LM step (``LMGen.step``, CUDA graph, 20 timed steps after 5) without and with cross-attention;
* ``cross_attn_step_kernel`` alone (``b200_op_cross_attn_step``, CUDA events) against its algorithmic bytes, the condition
  memory read once: ``2 * sessions * T * dim * 2`` per layer, as a share of the H100 SXM's 3.35 TB/s;
* ``LMGen.set_condition_cross`` of one session (every layer's K/V projection of its condition, outside the step).

Prints the card's name and power limit, then one JSON object per measurement.  Needs an 80 GB H100.

    python tools/cross_attention.py
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

DIM, HEADS, LAYERS, CONTEXT = 2048, 16, 16, 500
KEYS = (125, 625)
SESSIONS = (32, 64, 128, 256)
HBM_PEAK_GBS = 3350.0                   # H100 SXM data sheet (HBM3)
COND = {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 512}}}


def lm_kwargs(cross: bool) -> dict:
    import dataclasses

    from moshi_b200.config import LMConfig
    kw = dict(dim=DIM, num_heads=HEADS, num_layers=LAYERS, context=CONTEXT, text_card=8000, n_q=32, dep_q=16, card=2048,
              depformer_dim=1024, depformer_num_heads=16, depformer_num_layers=4, depformer_dim_feedforward=4224,
              depformer_context=16, delays=[0] + [2] * 32)
    if cross:
        kw.update(cross_attention=True, conditioners=COND, fuser={"cross": ["speaker_wavs"]})
    return dataclasses.asdict(LMConfig.from_dict(kw))


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


def conditions(lm, batch: int, keys: int):
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    g = torch.Generator().manual_seed(keys)
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(torch.randn(1, keys, 512, generator=g))})
             for _ in range(batch)]
    return lm.condition_provider(lm.condition_provider.prepare(attrs))


def lm_step(lm, batch: int, keys: int | None) -> dict:
    from moshi_b200.models import LMGen
    gen = LMGen(lm, condition_tensors=None if keys is None else conditions(lm, batch, keys))
    g = torch.Generator().manual_seed(1)
    codes = [torch.randint(0, 2048, (batch, 16, 1), generator=g).cuda() for _ in range(4)]
    out = {}
    with gen.streaming(batch), torch.no_grad():
        i = [0]

        def step():
            gen.step(codes[i[0] % 4])
            i[0] += 1
        out["step_ms"] = round(time_ms(step, 20), 3)
        if keys is not None:
            src = lm.fuser.get_cross(conditions(lm, 1, keys)).to(torch.bfloat16).cuda()
            out["set_condition_cross_one_session_ms"] = round(time_ms(lambda: gen.set_condition_cross(src, [0]), 20), 3)
    return out


def kernel(lib, batch: int, keys: int) -> dict:
    q = torch.randn(batch, HEADS * 128, device="cuda").bfloat16()
    k = torch.randn(batch, HEADS, keys, 128, device="cuda").bfloat16()
    v = torch.randn_like(k)
    out = torch.empty_like(q)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = time_ms(lambda: _lib.check(lib.b200_op_cross_attn_step(_lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(out), batch, HEADS,
                                                                keys, 0, s)), 200)
    nbytes = 2 * batch * keys * DIM * 2
    return {"kernel_us": round(ms * 1e3, 2), "algorithmic_bytes": nbytes, "gbs": round(nbytes / ms / 1e6, 1),
            "frac_of_hbm_peak": round(nbytes / ms / 1e6 / HBM_PEAK_GBS, 3)}


def main():
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi,
                      "geometry": {"dim": DIM, "heads": HEADS, "layers": LAYERS, "context": CONTEXT, "assumed": True}}), flush=True)
    lib = _lib.lib()
    for keys in KEYS:
        for batch in SESSIONS:
            print(json.dumps({"what": "cross_attn_step_kernel", "sessions": batch, "keys": keys, **kernel(lib, batch, keys)}), flush=True)
    torch.cuda.empty_cache()
    from moshi_b200.models import loaders
    for cross in (False, True):
        lm = loaders.get_moshi_lm(None, lm_kwargs(cross), device="cuda", synth_device="cuda")
        for batch in SESSIONS:
            for keys in (KEYS if cross else (None,)):
                print(json.dumps({"what": "lm_step", "cross_attention": cross, "sessions": batch, "keys": keys,
                                  **lm_step(lm, batch, keys)}), flush=True)
        del lm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
