#!/usr/bin/env python
"""Per-kernel micro-benchmarks (CUDA events) of the hot-path kernels through the C ABI.

Every timed launch reads operands that are not L2-resident: weights / KV rings are rotated through
enough copies to exceed the 126 MB L2.  Prints one JSON object per line; run under gpurun, e.g.

    python tools/kbench.py --what gemm,attn,mimi > gpurun_out/kbench.jsonl
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from moshi_b200 import _lib  # noqa: E402

PEAK = 6576.1
p = ROOT / "MEASURED_PEAKS.json"
if p.exists():
    PEAK = float(json.loads(p.read_text())["hbm_gbs"])


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def time_ms(fn, n_rot: int, iters: int = 20, warm: int = 3) -> float:
    for i in range(warm):
        fn(i % n_rot)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % n_rot)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_gemm(lib, Ms, legacy=True, only="", ns_sweep=False):
    shapes = [  # (name, N, K, epi, gate_rows)
        ("temporal.in_proj", 12288, 4096, 0, 0), ("temporal.out_proj", 4096, 4096, 1, 0),
        ("temporal.linear_in", 22528, 4096, 2, 11264), ("temporal.linear_out", 4096, 11264, 1, 0),
        ("text_linear", 32000, 4096, 0, 0), ("depformer_in_all", 8192, 4096, 0, 0),
        ("dep.in_proj", 3072, 1024, 0, 0), ("dep.out_proj", 1024, 1024, 1, 0), ("dep.linear_in", 5632, 1024, 2, 2816),
        ("dep.linear_out", 1024, 2816, 1, 0), ("dep.head", 2048, 1024, 0, 0),
    ]
    for name, N, K, epi, gr in shapes:
        if only and only not in name:
            continue
        wbytes = N * K * 2
        n_rot = max(2, -(-(400 << 20) // wbytes))
        ws = [torch.empty(N, K, device="cuda", dtype=torch.bfloat16).uniform_(-0.02, 0.02) for _ in range(n_rot)]
        pk = []
        for w in ws:
            out = torch.empty(lib.b200_op_packed_bytes(N, K, epi, gr), dtype=torch.uint8, device="cuda")
            _lib.check(lib.b200_op_pack_tiles(_lib.ptr(w), _lib.ptr(out), N, K, epi, gr, stream()))
            pk.append(out)
        cols = gr if epi == 2 else N
        for M in Ms:
            x = torch.empty(M, K, device="cuda", dtype=torch.bfloat16).uniform_(-1, 1)
            y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            res = torch.zeros(M, cols, device="cuda", dtype=torch.bfloat16)
            alg = wbytes + M * K * 2 + M * cols * 2 * (2 if epi == 1 else 1)
            # "lm": what the LM launches for this shape (GEMV <= 2 rows, swap-AB stream-K <= 32, non-swapped N=256 kernel 33..256);
            # "swapAB": the swap-AB kernels at any M; "ns.csN": the non-swapped kernel with K cut over N CTAs
            variants = [("lm", 0, 0, 0), ("swapAB", 0, -1, 0), ("swapAB.stream_only", 0, -1, 1)]
            if ns_sweep and M <= 128:
                n_units = -(-(gr if epi == 2 else N) // 128) if epi == 2 else -(-N // 256)
                variants += [(f"ns.cs{c}", -c, 0, 0) for c in ((1,) if epi == 2 else (1, 2, 3, 4, 8)) if n_units * c <= torch.cuda.get_device_properties(0).multi_processor_count]
                if epi != 2:
                    variants += [(f"ns.n128.cs{c}", -(100 + c), 0, 0) for c in (1, 2, 4) if -(-N // 128) * c <= torch.cuda.get_device_properties(0).multi_processor_count]
            for vname, grid, smem, so in variants:
                def fn(i):
                    if vname.startswith("ns."):
                        _lib.check(lib.b200_op_linear_ns(_lib.ptr(x), _lib.ptr(pk[i]), _lib.ptr(y), _lib.ptr(res), M, N, K, epi, gr,
                                                         -grid, stream()))
                    else:
                        _lib.check(lib.b200_op_linear_sk(_lib.ptr(x), _lib.ptr(pk[i]), _lib.ptr(y), _lib.ptr(res), M, N, K, epi, gr,
                                                         grid, smem, so, stream()))
                ms = time_ms(fn, n_rot)
                gbs = alg / ms / 1e6
                print(json.dumps({"kernel": "linear", "name": name, "M": M, "N": N, "K": K, "impl": vname, "ms": round(ms, 4),
                                  "GBps": round(gbs, 1), "frac": round(gbs / PEAK, 3)}), flush=True)
            if not legacy:
                continue
            # same-box library row: cuBLAS through torch.matmul on the row-major weights (the reference's path for every
            # nn.Linear, SURVEY 2b); GEMM only, i.e. without the residual add / gated SiLU our kernels fuse
            def fn(i):
                torch.matmul(x, ws[i].t())
            ms = time_ms(fn, n_rot)
            gbs = alg / ms / 1e6
            print(json.dumps({"kernel": "linear", "name": name, "M": M, "N": N, "K": K, "impl": "cublas(torch.matmul)", "ms": round(ms, 4),
                              "GBps": round(gbs, 1), "frac": round(gbs / PEAK, 3)}), flush=True)
        del ws, pk


def bench_attn(lib, Bs, cap=3000, H=32):
    for B in Bs:
        per = B * H * cap * 128 * 2
        n_rot = max(2, -(-(300 << 20) // (2 * per)))
        n_rot = min(n_rot, 8)
        ks = [torch.empty(B, H, cap, 128, device="cuda", dtype=torch.bfloat16).normal_() for _ in range(n_rot)]
        vs = [torch.empty(B, H, cap, 128, device="cuda", dtype=torch.bfloat16).normal_() for _ in range(n_rot)]
        q = torch.randn(B, 3 * H * 128, device="cuda").bfloat16()
        out = torch.empty(B, H * 128, device="cuda", dtype=torch.bfloat16)
        mask = torch.ones(B, dtype=torch.bool, device="cuda")
        for fill in (cap, cap // 4):
            offs = torch.full((B,), fill + 7 * cap if fill == cap else fill - 1, dtype=torch.int64, device="cuda")
            for ns in (0,):
                def fn(i):
                    _lib.check(lib.b200_op_attn_step(_lib.ptr(q), _lib.ptr(ks[i]), _lib.ptr(vs[i]), _lib.ptr(out),
                                                     _lib.ptr(offs), _lib.ptr(mask), B, H, cap, ns, 10000.0, stream()))
                ms = time_ms(fn, n_rot)
                alg = 2 * B * H * min(fill, cap) * 128 * 2
                gbs = alg / ms / 1e6
                print(json.dumps({"kernel": "attn_step", "B": B, "H": H, "cap": cap, "fill": fill, "nsplit": ns,
                                  "ms": round(ms, 4), "GBps": round(gbs, 1), "frac": round(gbs / PEAK, 3)}), flush=True)
        del ks, vs


def bench_attn_q8(lib, Bs, fmt, cap=3000, H=32):
    """The opt-in 8-bit rings' attention step (one byte per element + one fp32 scale per key row); fmt 1 = e4m3, 2 = int8."""
    for B in Bs:
        n_rot = 2
        ks = [torch.randint(0, 120, (B, H, cap, 128), device="cuda", dtype=torch.uint8) for _ in range(n_rot)]
        vs = [torch.randint(0, 120, (B, H, cap, 128), device="cuda", dtype=torch.uint8) for _ in range(n_rot)]
        sk = torch.full((B, H, cap), 0.01, device="cuda")
        sv = torch.full((B, H, cap), 0.01, device="cuda")
        q = torch.randn(B, 3 * H * 128, device="cuda").bfloat16()
        out = torch.empty(B, H * 128, device="cuda", dtype=torch.bfloat16)
        mask = torch.ones(B, dtype=torch.bool, device="cuda")
        for fill in (cap, cap // 4):
            offs = torch.full((B,), fill + 7 * cap if fill == cap else fill - 1, dtype=torch.int64, device="cuda")
            def fn(i):
                _lib.check(lib.b200_op_attn_step_q8(_lib.ptr(q), _lib.ptr(ks[i]), _lib.ptr(vs[i]), _lib.ptr(sk), _lib.ptr(sv), _lib.ptr(out),
                                                    _lib.ptr(offs), _lib.ptr(mask), B, H, cap, 0, 10000.0, fmt, stream()))
            ms = time_ms(fn, n_rot)
            alg = 2 * B * H * min(fill, cap) * (128 + 4)
            gbs = alg / ms / 1e6
            print(json.dumps({"kernel": "attn_step_f8" if fmt == 1 else "attn_step_i8", "B": B, "H": H, "cap": cap, "fill": fill, "ms": round(ms, 4),
                              "GBps": round(gbs, 1), "frac": round(gbs / PEAK, 3)}), flush=True)
        del ks, vs


def bench_mimi(Bs):
    from moshi_b200.models import loaders
    mimi = loaders.get_mimi(None, device="cuda", num_codebooks=8)
    for B in Bs:
        g = torch.Generator().manual_seed(1)
        pcm = (0.1 * torch.randn(B, 1, 1920, generator=g)).cuda()
        with mimi.streaming(B), torch.no_grad():
            codes = None
            for _ in range(260):      # fill both 250-slot transformer rings
                codes = mimi.encode(pcm)
                mimi.decode(codes)
            enc = time_ms(lambda i: mimi.encode(pcm), 1, iters=20)
            dec = time_ms(lambda i: mimi.decode(codes), 1, iters=20)
            alg = mimi.algorithmic_bytes()
        print(json.dumps({"kernel": "mimi", "B": B, "encode_ms": round(enc, 4), "decode_ms": round(dec, 4),
                          "frames_per_s": round(B * 1e3 / (enc + dec), 1), "alg_bytes": alg,
                          "GBps": round(alg / (enc + dec) / 1e6, 1),
                          "gflops": round(B * 0.9 / (enc + dec) * 1e3, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="gemm,attn,mimi")
    ap.add_argument("--M", default="1,16,96")
    ap.add_argument("--B", default="1,16,96")
    ap.add_argument("--only", default="", help="GEMM shape name filter")
    ap.add_argument("--no-legacy", action="store_true")
    ap.add_argument("--ns-sweep", action="store_true", help="time the non-swapped GEMM at every cluster size")
    args = ap.parse_args()
    lib = _lib.lib()
    torch.cuda.set_device(0)
    Ms = [int(v) for v in args.M.split(",")]
    Bs = [int(v) for v in args.B.split(",")]
    what = args.what.split(",")
    if "attn" in what:
        bench_attn(lib, Bs)
    if "attn_f8" in what:
        bench_attn_q8(lib, Bs, 1)
    if "attn_i8" in what:
        bench_attn_q8(lib, Bs, 2)
    if "gemm" in what:
        bench_gemm(lib, Ms, legacy=not args.no_legacy, only=args.only, ns_sweep=args.ns_sweep)
    if "mimi" in what:
        bench_mimi(Bs)


if __name__ == "__main__":
    main()
