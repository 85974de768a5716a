"""CPU: the launches the LM plans for its linears (b200_op_linear_plan: kernel, row blocks, grid, cluster, shared memory, stages
and every kernel parameter) equal tests/golden/linear_plans.json for every linear shape of the 7B, 2B, STT and TTS
geometries at M = 1..256, bf16 and int8, at 132 SMs and the default GEMV limit.  The table is written by
tools/gen_linear_plans.py; a change to it is a change of what the LM launches."""
import ctypes as C
import json
from pathlib import Path

import pytest

GOLDEN = Path(__file__).resolve().parent / "golden" / "linear_plans.json"


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    from moshi_b200.build import build
    build()
    return _lib.lib()


def _plan(lib, M, N, K, epi, gate_rows, norm, int8, sms, gemv, n_fields):
    from moshi_b200 import _lib
    cap = 2 + 4 * n_fields
    buf = (C.c_int64 * cap)()
    rc = lib.b200_op_linear_plan(M, N, K, epi, gate_rows, int8, norm, sms, gemv, buf, cap)
    assert rc == _lib.B200_OK, (M, N, K, epi, lib.b200_last_error())
    return int(buf[1]), [list(buf[2 + n_fields * i:2 + n_fields * (i + 1)]) for i in range(int(buf[0]))]


def test_plans_match_golden(lib):
    t = json.loads(GOLDEN.read_text())
    fields, rows = t["fields"], t["fields"].index("rows")
    keys = {",".join(map(str, v)) for v in t["shapes"].values()}
    assert {k.rsplit(",", 1)[0] for k in t["plans"]} == keys
    bad = []
    for k, runs in t["plans"].items():
        N, K, epi, gate_rows, norm, int8 = map(int, k.split(","))
        assert runs[0][0] == 1 and runs[-1][1] == t["max_m"] and all(a[1] + 1 == b[0] for a, b in zip(runs, runs[1:])), k
        for first, last, folded, blocks in runs:
            for M in range(first, last + 1):
                want = [list(b) for b in blocks]
                want[-1][rows] += M - first
                got = _plan(lib, M, N, K, epi, gate_rows, norm, int8, t["sms"], t["gemv_max_rows"], len(fields))
                if got != (folded, want):
                    bad.append((k, M, got, (folded, want)))
    assert not bad, bad[:5]


def test_plan_rejects_what_the_linear_rejects(lib):
    from moshi_b200 import _lib
    buf = (C.c_int64 * 80)()
    assert lib.b200_op_linear_plan(257, 4096, 4096, 0, 0, 0, 0, 132, 2, buf, 80) == _lib.B200_ERR_SHAPE     # more than 256 rows
    assert lib.b200_op_linear_plan(4, 4096, 4100, 0, 0, 0, 0, 132, 2, buf, 80) == _lib.B200_ERR_SHAPE      # K % 8
    assert lib.b200_op_linear_plan(64, 4096, 4104, 0, 0, 1, 0, 132, 2, buf, 80) == _lib.B200_ERR_SHAPE     # int8 K % 16
    assert lib.b200_op_linear_plan(4, 4096, 4096, 0, 0, 0, 0, 0, 2, buf, 80) == _lib.B200_ERR_INVALID      # no SMs
    assert lib.b200_op_linear_plan(4, 4096, 4096, 0, 0, 0, 0, 132, 2, buf, 10) == _lib.B200_ERR_INVALID    # no room
    # the norm folds exactly where the plan takes the GEMV: up to the GEMV limit
    for M, gemv, folded in ((2, 2, 1), (3, 2, 0), (3, 4, 1), (1, 0, 0)):
        assert lib.b200_op_linear_plan(M, 12288, 4096, 0, 0, 0, 1, 132, gemv, buf, 80) == _lib.B200_OK
        assert (buf[1], buf[2] == 1) == (folded, bool(folded)), (M, gemv)
