"""CPU: the plan runs of Mimi's tensor-core layers that tests/test_gpu_zz_mimi_plan_runs.py runs, and the per-output fp64 rule
it holds them to.

The runs are derived from b200_op_mimi_plan at the device's SM count (tests/util.py mimi_plan_runs); at 132 SMs they must
reproduce every run boundary and value of tests/golden/mimi_plans.json.

The rule of one 3xTF32 layer (tests/util.py tc_ratios: |got - want| <= tc_c(k-blocks per split) 2^-24 sum_k |a_k w_k|) must
accept fp32 emulations
of the kernel at every layer shape and every plan run of the golden table (2 sessions, the real K and the real K splits,
ragged last splits included): RNA rounding to tf32 by bit arithmetic, the three split products summed per 32-wide k-block,
the k-blocks per split and the splits in split order, everything in reverse, or one chain.  It must reject each of these
kernel bugs in every GEMM row (session, step) it touches: a lost k-block in the last split, a k-block counted in two splits,
one split's partial added twice, the last split dropped, a_lo * w_hi dropped (plain 2xTF32), a session group read one session
late, dilation ignored (on a dilated variant of encoder.4: the default configuration has no dilated layer), the carried
context taken from the neighbouring session or zero, and a transposed conv's x[t - 1] tap read from the frame instead of the
carry.

Every mutant is judged at every run under that run's constant.  The emulations need a constant of at most about 5.  The
narrowest mutant margin (the smallest, over the rows a mutant touches, of the row's worst ratio) is 2xTF32 at the deepest K,
encoder.12 (K = 8192) at 385..512 sessions (52 k-blocks per split, constant 81.6): 2.03.  TC_C and TC_CHAIN are pinned
below: loosening them fails this file.
"""
import json
from pathlib import Path

import pytest
import torch

from moshi_b200.config import MimiConfig
from tests.util import (TC_C, TC_CHAIN, TC_CONV, TC_CONVTR, mimi_plan_batches, mimi_plan_runs, mimi_tc_layers, tc_c, tc_op_shape,
                        tc_ratios, tc_ref64, tc_rows)

GOLDEN = json.loads((Path(__file__).resolve().parent / "golden" / "mimi_plans.json").read_text())
LAYERS = mimi_tc_layers(MimiConfig())
B = 2
_MARGINS: dict = {}


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    from moshi_b200.build import build
    build()
    return _lib.lib()


def test_plan_runs_reproduce_the_golden_table(lib):
    t = mimi_plan_runs(lib, GOLDEN["sms"], GOLDEN["max_b"])
    assert t["shapes"] == GOLDEN["shapes"]
    assert t["runs"] == GOLDEN["runs"]
    assert t["frame"] == GOLDEN["frame"]
    n = sum(len(r) for r in t["runs"].values())
    batches = mimi_plan_batches(lib, GOLDEN["sms"], GOLDEN["max_b"])
    print(f"{len(t['runs'])} layers, {n} layer runs, {len(t['frame'])} frame runs, {len(batches)} batches at run ends")
    assert (n, len(batches)) == (113, 58)


def test_layer_table_matches_the_plan():
    """mimi_tc_layers names the plan's layers and gives each the shape b200_op_mimi_plan reports."""
    assert list(LAYERS) == list(GOLDEN["shapes"])
    for name, v in GOLDEN["shapes"].items():
        assert tc_op_shape(LAYERS[name], v[-1]) == v[1:], name


def test_tc_c_is_pinned():
    """TC_C: 32 fp32 roundings of sum_k |a_k w_k| for chains of up to TC_CHAIN = 8 k-blocks, growing as the square root of
    longer chains (96 k-blocks: 111).  The fp32 emulations below need at most about 5; every mutant is rejected in every row
    it touches, the narrowest (2xTF32 at encoder.12, K = 8192, 52 k-blocks per split) by a factor of about 2."""
    assert TC_C <= 32.0 and TC_CHAIN >= 8
    assert tc_c(96) <= 32.0 * 12 ** 0.5 and tc_c(1) == TC_C


# ---- fp32 emulation of mimi_tc_kernel ---------------------------------------------------------------------------------------
def _tf32(x: torch.Tensor) -> torch.Tensor:
    """Round fp32 to tf32, to nearest with ties away from zero (cvt.rna.tf32.f32), by bit arithmetic."""
    return ((x.view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def _split(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    hi = _tf32(x)
    return hi, _tf32(x - hi)


def _elu32(x: torch.Tensor) -> torch.Tensor:
    return torch.where(x > 0, x, torch.expm1(x))


def _operands(layer: dict, ext: torch.Tensor, T: int, dil: int) -> tuple[torch.Tensor, torch.Tensor]:
    """The implicit GEMM's A [B T, K] (k = tap Cin + ci) over the extended activated input ext [B, Cin, P + T_in] (fp32), and
    the weight layout [N, K] of a weight given in the reference layout."""
    if layer["kind"] == TC_CONVTR:
        starts, step = [0, 1], 1
    else:
        starts, step = [j * dil for j in range(layer["k"])], layer["stride"]
    cols = [ext[:, :, s:s + (T - 1) * step + 1:step].permute(0, 2, 1) for s in starts]
    return torch.cat(cols, dim=-1).reshape(ext.shape[0] * T, -1)


def _weights_nk(layer: dict, w: torch.Tensor) -> torch.Tensor:
    if layer["kind"] == TC_CONVTR:
        S = layer["stride"]
        taps = torch.stack([w[:, :, S:], w[:, :, :S]], dim=-1).permute(2, 1, 0, 3)        # [S, Cout, Cin, 2]
        return taps.reshape(S * w.shape[1], w.shape[0], 2).permute(0, 2, 1).reshape(S * w.shape[1], -1)
    return w.permute(0, 2, 1).reshape(w.shape[0], -1)


def _block_partials(A: torch.Tensor, W: torch.Tensor, drop_lo_hi: bool = False) -> list[torch.Tensor]:
    """Per 32-wide k-block the fp32 sum of the split products, small terms first: (a_lo w_hi + a_hi w_lo) + a_hi w_hi."""
    ahi, alo = _split(A)
    whi, wlo = _split(W)
    out = []
    for k0 in range(0, A.shape[1], 32):
        s = slice(k0, k0 + 32)
        p = ahi[:, s] @ wlo[:, s].T
        if not drop_lo_hi:
            p = alo[:, s] @ whi[:, s].T + p
        out.append(p + ahi[:, s] @ whi[:, s].T)
    return out


def _reduce(parts: list[torch.Tensor], ksplit: int, kbps: int, order: str = "split", mutant: str | None = None) -> torch.Tensor:
    """The k-block partials summed as the kernel does at (ksplit, kb_per_split): each split's k-blocks [s kbps, min(num_kb,
    (s + 1) kbps)) in one fp32 chain, the split partials added in split order (order "split"); "reverse": blocks and splits in
    reverse; "chain": one chain over every block.  ``mutant``: a kernel bug of the split walk or of the reduction."""
    nkb = len(parts)
    splits = [list(range(s * kbps, min(nkb, (s + 1) * kbps))) for s in range(ksplit)] if order != "chain" else [list(range(nkb))]
    if mutant == "lost k-block in the last split":
        splits[-1] = splits[-1][:-1]
    elif mutant == "k-block counted twice":
        splits[-1] = [max(splits[-1][0] - 1, 0)] + splits[-1]
    seq = list(range(len(splits)))
    if mutant == "split partial added twice":
        seq.insert(0, len(splits) // 2)
    elif mutant == "last split dropped":
        seq = seq[:-1]
    if order == "reverse":
        splits = [s[::-1] for s in splits]
        seq = seq[::-1]
    part = []
    for blocks in splits:
        acc = torch.zeros_like(parts[0])
        for j in blocks:
            acc = acc + parts[j]
        part.append(acc)
    v = torch.zeros_like(parts[0])
    for s in seq:
        v = v + part[s]
    return v


def _to_ref_layout(layer: dict, y: torch.Tensor, T: int) -> torch.Tensor:
    """GEMM output [B T, N] -> [B, Cout, T'] (a transposed conv's row t holds steps t S .. t S + S - 1)."""
    Bn = y.shape[0] // T
    if layer["kind"] == TC_CONVTR:
        S, Co = layer["stride"], layer["cout"]
        return y.view(Bn, T, S, Co).permute(0, 3, 1, 2).reshape(Bn, Co, T * S)
    return y.view(Bn, T, -1).permute(0, 2, 1)


class Case:
    """One layer at B = 2 sessions: fp32 inputs, the fp64 reference and the fp32 emulation's pieces."""

    def __init__(self, name: str, layer: dict, T: int, seed: int):
        self.name, self.layer, self.T = name, layer, T
        g = torch.Generator().manual_seed(seed)
        tr = layer["kind"] == TC_CONVTR
        cin, cout, k, st, dil = layer["cin"], layer["cout"], layer["k"], layer["stride"], layer["dil"]
        self.S = st if tr else 1
        self.T_in = T if tr else T * st
        self.P = 1 if tr else (k - 1) * dil + 1 - st
        self.x = torch.randn(B, cin, self.T_in, generator=g)
        self.w = (torch.randn(cin, cout, k, generator=g) if tr else torch.randn(cout, cin, k, generator=g)) / (cin * k) ** 0.5
        self.bias = 0.5 * torch.randn(cout, generator=g)
        ctx = torch.randn(B, cin, self.P, generator=g)
        self.prev = _elu32(ctx) if layer["elu"] else ctx
        a = _elu32(self.x) if layer["elu"] else self.x
        self.ext = torch.cat([self.prev, a], dim=-1)
        self.W = _weights_nk(layer, self.w)
        self.want, self.scale = tc_ref64(TC_CONVTR if tr else TC_CONV, self.x, self.w, self.bias, self.prev, stride=st, dil=dil,
                                         elu=layer["elu"])
        self.parts = self.partials()

    def partials(self, ext: torch.Tensor | None = None, dil: int | None = None, drop_lo_hi: bool = False) -> list[torch.Tensor]:
        A = _operands(self.layer, self.ext if ext is None else ext, self.T, self.layer["dil"] if dil is None else dil)
        return _block_partials(A, self.W, drop_lo_hi)

    def output(self, v: torch.Tensor) -> torch.Tensor:
        b = self.bias.repeat(self.S) if self.layer["kind"] == TC_CONVTR else self.bias
        return _to_ref_layout(self.layer, v + b, self.T)

    def row_ratios(self, y: torch.Tensor, c: float) -> torch.Tensor:
        """Worst ratio of every GEMM row: [B, T]."""
        return tc_rows(tc_ratios(y, self.want, self.scale, c), self.layer["kind"], self.S).amax(-1)

    def need(self, y: torch.Tensor) -> float:
        return float(self.row_ratios(y, 1.0).max())


def _cases():
    out = []
    for i, (name, v) in enumerate(GOLDEN["shapes"].items()):
        out.append((name, LAYERS[name], v[-1], GOLDEN["runs"][name]))
    # the default configuration has no dilated layer: encoder.4 at dilation 2, on encoder.4's runs
    out.append(("encoder.4 dil 2", {**LAYERS["encoder.4"], "dil": 2}, GOLDEN["shapes"]["encoder.4"][-1], GOLDEN["runs"]["encoder.4"]))
    return out


CASES = _cases()
SPLIT_MUTANTS = ["lost k-block in the last split", "k-block counted twice", "split partial added twice", "last split dropped"]


def _reject(case: Case, y: torch.Tensor, rows: torch.Tensor, c: float, what: str) -> float:
    """Asserts that every GEMM row in ``rows`` ([B, T] bool) has an output outside the rule of constant c; returns the
    smallest such row's worst ratio (the mutant's margin)."""
    r = case.row_ratios(y, c)
    assert rows.any(), what
    admitted = (rows & (r <= 1)).nonzero().tolist()
    margin = float(r[rows].min())
    print(f"{what}: {int(rows.sum())} rows touched, margin {margin:.3g}")
    assert not admitted, (what, admitted[:8])
    _MARGINS[what] = margin
    return margin


def _input_mutants(case: Case, bb: int) -> list[tuple[str, list, torch.Tensor]]:
    """(name, k-block partials, GEMM rows touched) of the mutants that change what the kernel reads."""
    layer, T = case.layer, case.T
    every = torch.ones(B, T, dtype=torch.bool)
    out = [("a_lo w_hi dropped (2xTF32)", case.partials(drop_lo_hi=True), every)]
    # the first session group read one session late: its sessions see the next one's input, the last one zeros (TMA fill)
    late = torch.zeros_like(case.ext)
    late[:B - 1] = case.ext[1:]
    g0 = min(bb, B)
    ext = case.ext.clone()
    ext[:g0] = late[:g0]
    rows = torch.zeros(B, T, dtype=torch.bool)
    rows[:g0] = True
    out.append(("session group one session late", case.partials(ext=ext), rows))
    if layer["dil"] > 1:
        out.append(("dilation ignored", case.partials(dil=1), every))
    if case.P > 0:
        steps = torch.arange(T)
        ctx_rows = (steps == 0 if layer["kind"] == TC_CONVTR else steps * layer["stride"] < case.P)[None].expand(B, T)
        ext = case.ext.clone()
        ext[:, :, :case.P] = case.ext[[1, 0], :, :case.P]
        out.append(("carried context of the neighbouring session", case.partials(ext=ext), ctx_rows))
        ext = case.ext.clone()
        ext[:, :, :case.P] = 0
        out.append(("carried context zero", case.partials(ext=ext), ctx_rows))
        if layer["kind"] == TC_CONVTR:
            ext = case.ext.clone()
            ext[:, :, 0] = case.ext[:, :, 1]
            out.append(("x[t - 1] tap read from the frame instead of the carry", case.partials(ext=ext), ctx_rows))
    return out


@pytest.mark.parametrize("name,layer,T,runs", CASES, ids=[c[0] for c in CASES])
def test_rule_accepts_every_plan_run_and_rejects_every_mutant(name, layer, T, runs):
    case = Case(name, layer, T, seed=len(name) * 131 + T)
    nkb = len(case.parts)
    needs = []
    mutants = None
    every = torch.ones(B, T, dtype=torch.bool)
    for first, last, f in runs:
        bb, ksplit, kbps = f[1], f[2], f[3]
        c = tc_c(kbps)
        for order in ("split", "reverse", "chain"):
            y = case.output(_reduce(case.parts, ksplit, kbps, order))
            needs.append(case.need(y))
            assert case.need(y) <= (tc_c(nkb) if order == "chain" else c), (name, first, last, order, case.need(y))
        run = f"{name} run {first}-{last} ({ksplit} x {kbps} over {nkb}, constant {c:.3g})"
        for m in SPLIT_MUTANTS:
            if ksplit == 1 and m in ("split partial added twice", "last split dropped"):
                continue
            _reject(case, case.output(_reduce(case.parts, ksplit, kbps, mutant=m)), every, c, f"{run}: {m}")
        mutants = mutants or _input_mutants(case, bb)
        for m, parts, rows in mutants:
            _reject(case, case.output(_reduce(parts, ksplit, kbps)), rows, c, f"{run}: {m}")
    print(f"{name}: {len(runs)} runs, largest constant needed {max(needs):.3g}")


def test_zz_narrowest_margin():
    """Prints the narrowest mutant margins of the run above (on a run of the whole file)."""
    if not _MARGINS:
        pytest.skip("no mutant ran")
    worst = sorted(_MARGINS.items(), key=lambda kv: kv[1])[:5]
    print("narrowest margins: " + "; ".join(f"{k} {v:.3g}" for k, v in worst))
    assert worst[0][1] > 1
