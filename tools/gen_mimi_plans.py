"""Writes tests/golden/mimi_plans.json: what Mimi launches per frame at 1..512 sessions for the default MimiConfig on 132 SMs
(H100 SXM), as b200_op_mimi_plan reports it.  Needs the built library, no GPU.

Per tensor-core layer (both SEANets, then the four transformer linears, which serve every layer of both transformers) its
static shape, then runs [B_first, B_last, schedule] over which the schedule (FIELDS) is constant; the row tiles and the grid
follow from it (tests/test_mimi_plans_cpu.py checks that rule).  "frame" holds the runs of the per-frame values (FRAME): the
down-sampling conv's K slices, the split-K workspace bytes and the kernels of one encode and one decode frame.

    python tools/gen_mimi_plans.py          # rewrite the golden
"""
from __future__ import annotations

import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from moshi_b200 import _lib  # noqa: E402
from moshi_b200.config import MimiConfig  # noqa: E402
from moshi_b200.models.compression import _config_struct  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "mimi_plans.json"
SMS, MAX_B, CAPACITY = 132, 512, 1024
HEAD = ["enc_layers", "dec_layers", "down_ksplit", "ws_bytes", "enc_launches", "dec_launches"]
LAYER = ["layer", "kind", "Cin", "N", "n_taps", "dil", "stride", "NT", "n_tiles_n", "num_kb", "tt", "bb", "T", "n_sessions",
         "m_tiles", "ksplit", "kb_per_split", "stages", "stage_bytes", "grid", "smem"]
SHAPE = ["kind", "Cin", "N", "n_taps", "dil", "stride", "NT", "n_tiles_n", "num_kb", "T"]
FIELDS = ["tt", "bb", "ksplit", "kb_per_split", "stages", "stage_bytes", "smem", "NT"]
FRAME = ["down_ksplit", "ws_bytes", "enc_launches", "dec_launches"]
LINEARS = ["in_proj", "out_proj", "linear1", "linear2"]


def plan(B: int, sms: int = SMS, num_codebooks: int | None = None, cfg: MimiConfig | None = None,
         capacity: int = CAPACITY, lib=None) -> tuple[int, dict, dict[str, dict]]:
    """(return code, header by HEAD, {layer name: values by LAYER}) of b200_op_mimi_plan (``lib``: the loaded library)."""
    cfg = cfg or MimiConfig()
    buf = (C.c_int64 * capacity)()
    c = _config_struct(cfg)
    ncb = cfg.num_codebooks if num_codebooks is None else num_codebooks
    rc = (lib or _lib.lib()).b200_op_mimi_plan(C.byref(c), B, sms, ncb, buf, capacity)
    if rc != _lib.B200_OK:
        return rc, {}, {}
    head = dict(zip(HEAD, buf[:len(HEAD)]))
    n_enc, n_dec = head["enc_layers"], head["dec_layers"]
    layers = {}
    for i in range(n_enc + n_dec + len(LINEARS)):
        v = dict(zip(LAYER, buf[len(HEAD) + len(LAYER) * i:len(HEAD) + len(LAYER) * (i + 1)]))
        name = (f"encoder.{v['layer']}" if i < n_enc else f"decoder.{v['layer']}" if i < n_enc + n_dec
                else f"transformer.{LINEARS[i - n_enc - n_dec]}")
        layers[name] = v
    return rc, head, layers


def add_run(runs: list[list], B: int, value: list[int]) -> None:
    if runs and runs[-1][2] == value:
        runs[-1][1] = B
    else:
        runs.append([B, B, value])


def plan_runs(sms: int = SMS, max_b: int = MAX_B, lib=None) -> tuple[dict[str, list[int]], dict[str, list[list]], list[list]]:
    """(SHAPE per layer, runs [B_first, B_last, FIELDS] per layer, runs [B_first, B_last, FRAME]) over 1..max_b sessions."""
    shapes: dict[str, list[int]] = {}
    runs: dict[str, list[list]] = {}
    frame: list[list] = []
    for B in range(1, max_b + 1):
        rc, head, layers = plan(B, sms, lib=lib)
        assert rc == _lib.B200_OK, (B, rc)
        add_run(frame, B, [head[f] for f in FRAME])
        for name, v in layers.items():
            shape = [v[f] for f in SHAPE]
            assert shapes.setdefault(name, shape) == shape, (name, B)
            add_run(runs.setdefault(name, []), B, [v[f] for f in FIELDS])
    return shapes, runs, frame


def table() -> dict:
    shapes, runs, frame = plan_runs()
    return {"sms": SMS, "max_b": MAX_B, "shape_fields": SHAPE, "fields": FIELDS, "frame_fields": FRAME, "frame": frame,
            "shapes": shapes, "runs": runs}


def dump(t: dict) -> str:
    """One line per run: reviewable in a diff."""
    lines = ["{", f' "sms": {t["sms"]}, "max_b": {t["max_b"]},', f' "shape_fields": {json.dumps(t["shape_fields"])},',
             f' "fields": {json.dumps(t["fields"])},', f' "frame_fields": {json.dumps(t["frame_fields"])},', ' "frame": [']
    lines += ["  " + json.dumps(r, separators=(",", ":")) + ("," if j + 1 < len(t["frame"]) else "") for j, r in enumerate(t["frame"])]
    lines += [" ],", ' "shapes": {']
    items = list(t["shapes"].items())
    lines += [f'  {json.dumps(n)}: {json.dumps(v)}' + ("," if i + 1 < len(items) else "") for i, (n, v) in enumerate(items)]
    lines += [" },", ' "runs": {']
    keys = list(t["runs"])
    for i, k in enumerate(keys):
        runs = t["runs"][k]
        lines.append(f'  {json.dumps(k)}: [')
        lines += ["   " + json.dumps(r, separators=(",", ":")) + ("," if j + 1 < len(runs) else "") for j, r in enumerate(runs)]
        lines.append("  ]" + ("," if i + 1 < len(keys) else ""))
    lines += [" }", "}"]
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    GOLDEN.write_text(dump(table()))
    print(f"wrote {GOLDEN}")
