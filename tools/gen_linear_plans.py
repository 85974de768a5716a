"""Writes tests/golden/linear_plans.json: the launches the LM plans for every linear shape it runs (b200_op_linear_plan), at
132 SMs (H100 SXM) and the default GEMV limit of 2 rows, for M = 1..256, bf16 and int8.  Needs the built library, no GPU.

Shapes: the 7B model's temporal in_proj, out_proj, gated linear_in, linear_out, text head and stacked depformer_in, and the
depformer chain's four linears and its heads; the same for the 2B model (tests/golden/moshi_dev_2b.json) and the STT geometry
of tests/test_gpu_zz_temporal_ref.py; the cross-attention q / K|V / out linears at the TTS geometry of
tests/test_gpu_zz_cross_ref.py.  The linears behind an RMSNorm (in_proj, linear_in) are planned with the norm, as norm_linear
asks for them.

Stored compactly: per distinct (N, K, epi, gate_rows, norm, int8) a list of runs [M_first, M_last, norm_folded, launches], the
launches being those of M_first (FIELDS per launch); within a run only the last launch's row count grows with M.

    python tools/gen_linear_plans.py          # rewrite the golden
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

GOLDEN = ROOT / "tests" / "golden" / "linear_plans.json"
SMS, GEMV_MAX_ROWS, MAX_M = 132, 2, 256
FIELDS = ["kernel", "m0", "rows", "grid", "cluster", "smem", "stages", "stage_bytes", "np", "Mpad", "kb_per", "S", "kbps",
          "unit_tiles", "ldw", "Wc", "whole_rounds", "sk_tile0", "sk_items"]
STORE, RESADD, GATE = 0, 1, 2


def _configs() -> dict[str, LMConfig]:
    two_b = LMConfig.from_dict(json.loads((ROOT / "tests" / "golden" / "moshi_dev_2b.json").read_text()))
    stt = LMConfig(dim=2048, num_heads=16, num_layers=4, n_q=32, dep_q=0, text_card=8000, delays=[0] * 33, extra_heads_num_heads=4,
                   extra_heads_dim=6)
    return {"7b": MOSHI_7B, "2b": two_b, "stt": stt}


def shapes() -> dict[str, tuple[int, int, int, int, int]]:
    """name -> (N, K, epi, gate_rows, norm) of every linear the LM launches."""
    out = {}
    for name, c in _configs().items():
        d, F = c.dim, c.ffn_hidden
        out[f"{name}.in_proj"] = (3 * d, d, STORE, 0, 1)
        out[f"{name}.out_proj"] = (d, d, RESADD, 0, 0)
        out[f"{name}.linear_in"] = (2 * F, d, GATE, F, 1)
        out[f"{name}.linear_out"] = (d, F, RESADD, 0, 0)
        out[f"{name}.text_linear"] = (c.text_card, d, STORE, 0, 0)
        if c.dep_q:
            dd, dF = c.depformer_dim, c.depformer_ffn_hidden
            out[f"{name}.depformer_in"] = (c.dep_q * dd, d, STORE, 0, 0)
            out[f"{name}.dep.in_proj"] = (3 * dd, dd, STORE, 0, 1)
            out[f"{name}.dep.out_proj"] = (dd, dd, RESADD, 0, 0)
            out[f"{name}.dep.linear_in"] = (2 * dF, dd, GATE, dF, 1)
            out[f"{name}.dep.linear_out"] = (dd, dF, RESADD, 0, 0)
            out[f"{name}.dep.head"] = (c.card, dd, STORE, 0, 0)
    d = 2048                                       # the TTS member of tests/test_gpu_zz_cross_ref.py (bf16 only)
    out["tts.cross.q"] = (d, d, STORE, 0, 0)
    out["tts.cross.kv"] = (2 * d, d, STORE, 0, 0)
    out["tts.cross.out"] = (d, d, RESADD, 0, 0)
    return out


def key(N: int, K: int, epi: int, gate_rows: int, norm: int, int8: int) -> str:
    return f"{N},{K},{epi},{gate_rows},{norm},{int8}"


def plan(M: int, N: int, K: int, epi: int, gate_rows: int, norm: int, int8: int) -> tuple[int, int, list[list[int]]]:
    """(return code, norm folded, launches) of b200_op_linear_plan."""
    cap = 2 + 4 * len(FIELDS)
    buf = (C.c_int64 * cap)()
    rc = _lib.lib().b200_op_linear_plan(M, N, K, epi, gate_rows, int8, norm, SMS, GEMV_MAX_ROWS, buf, cap)
    if rc != _lib.B200_OK:
        return rc, 0, []
    n = len(FIELDS)
    return rc, int(buf[1]), [list(buf[2 + n * i:2 + n * (i + 1)]) for i in range(int(buf[0]))]


def expand(first: list[list[int]], dm: int) -> list[list[int]]:
    """The launches of M_first + dm within a run: the last launch has dm more rows."""
    out = [list(b) for b in first]
    out[-1][FIELDS.index("rows")] += dm
    return out


def runs_for(N: int, K: int, epi: int, gate_rows: int, norm: int, int8: int) -> list[list]:
    runs: list[list] = []
    for M in range(1, MAX_M + 1):
        rc, folded, blocks = plan(M, N, K, epi, gate_rows, norm, int8)
        assert rc == _lib.B200_OK, (N, K, epi, M, rc)
        if runs:
            r = runs[-1]
            if r[1] == M - 1 and r[2] == folded and len(r[3]) == len(blocks) and expand(r[3], M - r[0]) == blocks:
                r[1] = M
                continue
        runs.append([M, M, folded, blocks])
    return runs


def table() -> dict:
    sh = shapes()
    plans = {}
    for name, (N, K, epi, gr, norm) in sh.items():
        for int8 in ((0,) if name.startswith("tts.") else (0, 1)):
            k = key(N, K, epi, gr, norm, int8)
            if k not in plans:
                plans[k] = runs_for(N, K, epi, gr, norm, int8)
    return {"sms": SMS, "gemv_max_rows": GEMV_MAX_ROWS, "max_m": MAX_M, "fields": FIELDS,
            "shapes": {n: list(v) for n, v in sh.items()}, "plans": plans}


def dump(t: dict) -> str:
    """One line per run: reviewable in a diff."""
    lines = ["{", f' "sms": {t["sms"]}, "gemv_max_rows": {t["gemv_max_rows"]}, "max_m": {t["max_m"]},',
             f' "fields": {json.dumps(t["fields"])},', ' "shapes": {']
    items = list(t["shapes"].items())
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
