"""CPU: the depformer path the LM plans at streaming_begin and the persistent kernel's schedule (b200_op_depformer_plan) equal
tests/golden/depformer_plans.json for the 7B, 2B, q16, ragged and STT geometries at 1..256 sessions (1..128 under
classifier-free guidance), guidance and int8 on and off, every b200_lm_set_depformer mode and GEMV limits 2 and 4, at 132 SMs.
The table is written by tools/gen_depformer_plans.py; a change to it is a change of what the LM launches."""
import ctypes as C
import json
from pathlib import Path

import pytest

GOLDEN = Path(__file__).resolve().parent / "golden" / "depformer_plans.json"
NONE, CHAIN, FUSED = 0, 1, 2


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    from moshi_b200.build import build
    build()
    return _lib.lib()


def _plan(lib, geom, B, cfg, int8, mode, sms, gemv, n=36):
    buf = (C.c_int64 * n)()
    rc = lib.b200_op_depformer_plan(*geom, B, cfg, int8, mode, sms, gemv, buf, n)
    return rc, list(buf)


def test_plans_match_golden(lib):
    from moshi_b200 import _lib
    t = json.loads(GOLDEN.read_text())
    n = len(t["fields"])
    keys = {k.split(",", 5)[5] for k in t["plans"]}
    assert keys == {f"{c},{i},{m},{g}" for c in (0, 1) for i in (0, 1) for m in (0, 1, 2) for g in (2, 4)}
    assert {",".join(map(str, g)) for g in t["geometries"].values()} == {k.rsplit(",", 4)[0] for k in t["plans"]}
    bad = []
    for k, runs in t["plans"].items():
        v = list(map(int, k.split(",")))
        geom, (cfg, int8, mode, gemv) = v[:5], v[5:]
        top = t["max_b"] // 2 if cfg else t["max_b"]
        assert runs[0][0] == 1 and runs[-1][1] == top and all(a[1] + 1 == b[0] for a, b in zip(runs, runs[1:])), k
        for first, last, p in runs:
            for B in range(first, last + 1):
                want = list(p)
                want[1] = p[1] // first * B
                rc, got = _plan(lib, geom, B, cfg, int8, mode, t["sms"], gemv, n)
                if rc != _lib.B200_OK or got != want:
                    bad.append((k, B, rc, got[:6], want[:6]))
    assert not bad, bad[:5]


def test_path_rules(lib):
    """The persistent kernel runs from three sessions on (from one when forced), never under guidance, with int8 linears or in
    chain mode; no depformer plans none in every mode."""
    g7 = (8, 1024, 16, 2816, 2048)
    for B, cfg, int8, mode, gemv, path in ((2, 0, 0, 0, 2, CHAIN), (3, 0, 0, 0, 2, FUSED), (4, 0, 0, 0, 4, CHAIN), (1, 0, 0, 2, 2, FUSED),
                                           (3, 1, 0, 2, 2, CHAIN), (3, 0, 1, 2, 2, CHAIN), (256, 0, 0, 1, 2, CHAIN)):
        rc, p = _plan(lib, g7, B, cfg, int8, mode, 132, gemv)
        assert rc == 0 and p[0] == path, (B, cfg, int8, mode, gemv, p[0])
    for mode in (0, 1, 2):
        assert _plan(lib, (0, 1024, 16, 2816, 2048), 3, 0, 0, mode, 132, 2)[1][0] == NONE
    # depformer_dim above the row phases' reach or not a multiple of 64: the launch chain
    assert _plan(lib, (8, 1088, 17, 2816, 2048), 3, 0, 0, 2, 132, 2)[1][0] == CHAIN
    assert _plan(lib, (8, 992, 16, 2816, 2048), 3, 0, 0, 2, 132, 2)[1][0] == CHAIN


def test_plan_rejects_out_of_range(lib):
    from moshi_b200 import _lib
    g7 = (8, 1024, 16, 2816, 2048)
    INV = _lib.B200_ERR_INVALID
    assert _plan(lib, g7, 0, 0, 0, 0, 132, 2)[0] == INV           # no session
    assert _plan(lib, g7, 257, 0, 0, 0, 132, 2)[0] == INV         # more than 256 model rows
    assert _plan(lib, g7, 129, 1, 0, 0, 132, 2)[0] == INV         # 258 model rows under guidance
    assert _plan(lib, g7, 3, 0, 0, 3, 132, 2)[0] == INV           # unknown mode
    assert _plan(lib, g7, 3, 0, 0, 0, 0, 2)[0] == INV             # no SMs
    assert _plan(lib, g7, 3, 0, 0, 0, 132, 5)[0] == INV           # GEMV limit past 4 rows
    assert _plan(lib, (17, 1024, 16, 2816, 2048), 3, 0, 0, 0, 132, 2)[0] == INV   # dep_q past 16
    assert _plan(lib, g7, 3, 0, 0, 0, 132, 2, n=35)[0] == INV     # no room
    # a configuration the persistent kernel cannot run (head dim 128, ffn not a multiple of 8) is refused where the plan takes
    # it, and runs as the launch chain
    for geom in ((8, 1024, 8, 2816, 2048), (8, 1024, 16, 2820, 2048)):
        assert _plan(lib, geom, 3, 0, 0, 0, 132, 2)[0] == INV
        assert _plan(lib, geom, 3, 0, 0, 1, 132, 2)[0] == _lib.B200_OK
