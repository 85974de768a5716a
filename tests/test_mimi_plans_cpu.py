"""CPU: what Mimi launches per frame (b200_op_mimi_plan, the plan b200_mimi_streaming_begin binds) equals
tests/golden/mimi_plans.json for the default MimiConfig at 1..512 sessions on 132 SMs: every tensor-core layer's shape and
schedule, the down-sampling conv's K slices, the split-K workspace and the kernels of one encode and one decode frame.
The table is written by tools/gen_mimi_plans.py; a change to it is a change of what Mimi launches."""
import ctypes as C
import json
import sys
from dataclasses import replace
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "mimi_plans.json"


@pytest.fixture(scope="module")
def gen():
    from moshi_b200.build import build
    build()
    sys.path.insert(0, str(ROOT / "tools"))
    import gen_mimi_plans
    return gen_mimi_plans


def test_plans_match_golden(gen):
    t = json.loads(GOLDEN.read_text())
    assert (t["sms"], t["max_b"], t["fields"], t["frame_fields"]) == (gen.SMS, gen.MAX_B, gen.FIELDS, gen.FRAME)
    for runs in [t["frame"], *t["runs"].values()]:
        assert runs[0][0] == 1 and runs[-1][1] == t["max_b"] and all(a[1] + 1 == b[0] for a, b in zip(runs, runs[1:]))
    bad = []
    for B in range(1, t["max_b"] + 1):
        rc, head, layers = gen.plan(B, t["sms"])
        assert rc == 0, B
        frame = next(v for b0, b1, v in t["frame"] if b0 <= B <= b1)
        if [head[f] for f in gen.FRAME] != frame:
            bad.append(("frame", B))
        assert list(layers) == list(t["runs"]), B
        for name, v in layers.items():
            want = next(p for b0, b1, p in t["runs"][name] if b0 <= B <= b1)
            if [v[f] for f in gen.SHAPE] != t["shapes"][name] or [v[f] for f in gen.FIELDS] != want:
                bad.append((name, B))
    assert not bad, bad[:5]


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_tiling_contract(gen, sms):
    """The kernel's tile walk (tile_at): m_tiles = ceil(T / tt) * ceil(B / bb) row tiles of tt * bb = 128 rows, a grid of at most
    one CTA per tile and split; the TMA box of tt * stride rows stays within 256; K splits cover the k-blocks."""
    for B in (1, 2, 3, 7, 16, 63, 64, 65, 100, 128, 129, 200, 256, 300, 512):
        rc, head, layers = gen.plan(B, sms)
        assert rc == 0
        assert head["ws_bytes"] >= 64 << 20
        for name, v in layers.items():
            tt, bb, T, ks = v["tt"], v["bb"], v["T"], v["ksplit"]
            assert v["n_sessions"] == B and tt * bb == 128 and tt * v["stride"] <= 256 and T % tt == 0, (name, B, v)
            assert v["m_tiles"] == -(-T // tt) * -(-B // bb), (name, B)
            assert v["grid"] == min(v["m_tiles"] * v["n_tiles_n"] * ks, sms), (name, B)
            assert ks == -(-v["num_kb"] // v["kb_per_split"]) and (ks - 1) * v["kb_per_split"] < v["num_kb"], (name, B)
            if ks > 1:
                assert ks * v["m_tiles"] * 128 * v["N"] * 4 <= 64 << 20, (name, B)


def test_launch_counts_follow_codebooks(gen):
    """Each active codebook level past the first adds one search and one pick launch to an encode frame; decode is unchanged."""
    _, h8, _ = gen.plan(4, num_codebooks=8)
    _, h16, _ = gen.plan(4, num_codebooks=16)
    assert h16["enc_launches"] - h8["enc_launches"] == 16 and h16["dec_launches"] == h8["dec_launches"]


def test_plan_rejects_out_of_range(gen):
    from moshi_b200 import _lib
    from moshi_b200.config import MimiConfig
    INV = _lib.B200_ERR_INVALID
    assert gen.plan(1)[0] == _lib.B200_OK
    assert gen.plan(0)[0] == INV                                        # no session
    assert gen.plan(4, sms=0)[0] == INV                                 # no SMs
    assert gen.plan(4, num_codebooks=0)[0] == INV                       # fewer codebooks than the semantic ones
    assert gen.plan(4, num_codebooks=33)[0] == INV                      # more than the checkpoint holds
    assert gen.plan(4, capacity=6 + 21 * 30 - 1)[0] == INV              # no room
    assert gen.plan(4, capacity=6 + 21 * 30)[0] == _lib.B200_OK
    # configurations b200_mimi_create refuses
    for bad in (dict(channels=2), dict(n_filters=48), dict(tr_num_heads=4), dict(frame_rate=12.0), dict(ratios=[8, 6, 5, 3])):
        assert gen.plan(4, cfg=replace(MimiConfig(), **bad))[0] == INV, bad
    assert _lib.lib().b200_op_mimi_plan(None, 4, 132, 8, (C.c_int64 * 1024)(), 1024) == INV
