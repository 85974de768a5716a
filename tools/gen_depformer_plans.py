"""Writes tests/golden/depformer_plans.json: the depformer path the LM plans at streaming_begin (b200_op_depformer_plan) and, for
the persistent kernel, its schedule: partial-buffer floats, stages, shared memory, grid and the five GEMM phases' splits.  At 132
SMs (H100 SXM) and GEMV limits of 2 (the default) and 4 rows, for 1..256 sessions (1..128 under classifier-free guidance, which
doubles the model rows), guidance on and off, int8 linears on and off, and every b200_lm_set_depformer mode.  Needs the built
library, no GPU.

Geometries: the 7B and 2B models (tests/golden/moshi_dev_2b.json), the "q16" and "ragged" members of
tests/test_gpu_zz_depformer_ref.py and the STT geometry (dep_q = 0: no depformer).

Stored compactly: per distinct (dep_q, dd, heads, ffn, card, cfg, int8, mode, gemv rows) a list of runs [B_first, B_last,
plan], the plan being that of B_first (FIELDS); within a run only the partial-buffer floats change, in proportion to B.

    python tools/gen_depformer_plans.py          # rewrite the golden
"""
from __future__ import annotations

import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from moshi_b200 import _lib  # noqa: E402
from moshi_b200.config import MOSHI_7B, LMConfig  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "depformer_plans.json"
SMS, GEMV_MAX_ROWS, MAX_B = 132, (2, 4), 256
PHASES = ["in_proj", "out_proj", "linear_in", "linear_out", "head"]
FIELDS = ["path", "part_floats", "stages", "stage_bytes", "smem", "grid"] + [
    f"{p}.{f}" for p in PHASES for f in ("n_tiles", "num_kb", "kbps", "S", "A", "N")]
MODES = (_lib.B200_DEPFORMER_AUTO, _lib.B200_DEPFORMER_CHAIN, _lib.B200_DEPFORMER_FUSED)


def geometries() -> dict[str, tuple[int, int, int, int, int]]:
    """name -> (dep_q, depformer_dim, depformer_num_heads, depformer_ffn_hidden, card)."""
    two_b = LMConfig.from_dict(json.loads((ROOT / "tests" / "golden" / "moshi_dev_2b.json").read_text()))
    q16 = LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=4000, n_q=32, dep_q=16, depformer_context=16,
                   depformer_num_layers=2, delays=[0, 0] + [2] * 15 + [0] + [2] * 15)
    ragged = LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=1000, card=1000, depformer_dim=512,
                      depformer_num_heads=8, depformer_dim_feedforward=1500, depformer_num_layers=2)
    stt = LMConfig(dim=2048, num_heads=16, num_layers=4, n_q=32, dep_q=0, text_card=8000, delays=[0] * 33, extra_heads_num_heads=4,
                   extra_heads_dim=6)
    cfgs = {"7b": MOSHI_7B, "2b": two_b, "q16": q16, "ragged": ragged, "stt": stt}
    return {n: (c.dep_q, c.depformer_dim, c.depformer_num_heads, c.depformer_ffn_hidden, c.card) for n, c in cfgs.items()}


def key(geom: tuple[int, ...], cfg: int, int8: int, mode: int, gemv: int) -> str:
    return ",".join(map(str, (*geom, cfg, int8, mode, gemv)))


def plan(geom: tuple[int, ...], B: int, cfg: int, int8: int, mode: int, gemv: int, sms: int = SMS) -> tuple[int, list[int]]:
    """(return code, FIELDS) of b200_op_depformer_plan."""
    buf = (C.c_int64 * len(FIELDS))()
    rc = _lib.lib().b200_op_depformer_plan(*geom, B, cfg, int8, mode, sms, gemv, buf, len(FIELDS))
    return rc, list(buf) if rc == _lib.B200_OK else []


def expand(first: list[int], b0: int, B: int) -> list[int]:
    """The plan of B within a run that starts at b0 with plan `first`: the partial buffers grow with B."""
    out = list(first)
    out[1] = first[1] // b0 * B
    return out


def runs_for(geom: tuple[int, ...], cfg: int, int8: int, mode: int, gemv: int) -> list[list]:
    runs: list[list] = []
    for B in range(1, (MAX_B // 2 if cfg else MAX_B) + 1):
        rc, p = plan(geom, B, cfg, int8, mode, gemv)
        assert rc == _lib.B200_OK, (geom, B, cfg, int8, mode, gemv, rc)
        if runs and expand(runs[-1][2], runs[-1][0], B) == p:
            runs[-1][1] = B
        else:
            runs.append([B, B, p])
    return runs


def table() -> dict:
    geoms = geometries()
    plans = {}
    for geom in geoms.values():
        for cfg in (0, 1):
            for int8 in (0, 1):
                for mode in MODES:
                    for gemv in GEMV_MAX_ROWS:
                        k = key(geom, cfg, int8, mode, gemv)
                        if k not in plans:
                            plans[k] = runs_for(geom, cfg, int8, mode, gemv)
    return {"sms": SMS, "max_b": MAX_B, "fields": FIELDS, "geometries": {n: list(g) for n, g in geoms.items()}, "plans": plans}


def dump(t: dict) -> str:
    """One line per run: reviewable in a diff."""
    lines = ["{", f' "sms": {t["sms"]}, "max_b": {t["max_b"]},', f' "fields": {json.dumps(t["fields"])},', ' "geometries": {']
    items = list(t["geometries"].items())
    lines += [f'  {json.dumps(n)}: {json.dumps(v)}' + ("," if i + 1 < len(items) else "") for i, (n, v) in enumerate(items)]
    lines += [" },", ' "plans": {']
    keys = list(t["plans"])
    for i, k in enumerate(keys):
        runs = t["plans"][k]
        lines.append(f'  {json.dumps(k)}: [')
        lines += ["   " + json.dumps(r, separators=(",", ":")) + ("," if j + 1 < len(runs) else "") for j, r in enumerate(runs)]
        lines.append("  ]" + ("," if i + 1 < len(keys) else ""))
    lines += [" }", "}"]
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    GOLDEN.write_text(dump(table()))
    print(f"wrote {GOLDEN}")
