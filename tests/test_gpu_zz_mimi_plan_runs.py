"""GPU: every tensor-core layer of Mimi at both ends of each of its plan runs, against float64.

The runs come from b200_op_mimi_plan at this device's SM count (tests/util.py mimi_plan_runs), so a change of plan_tc or
plan_mimi moves the tested batches with it.  For every layer and every run, b200_op_tc_conv1d runs at the run's first and
last session count with the layer's own geometry (tests/util.py mimi_tc_layers: Cin, Cout, taps, stride, dilation, steps and
the ELU on the input; the transformer linears as 1-tap convs over their 2 steps, which plan_tc schedules as it does the
linears).  The op plans through the same plan_tc on the same SM count and split-K budget; the test asserts that the shape it
hands plan_tc is the one the plan reports for the layer, so it cannot silently test another schedule.

Each case runs two chunks from a random carried context; in the second one session at a group edge is paused.  Checked on
every session and output: both chunks within the fp64 rule (tests/util.py tc_ratios <= 1 under tc_c of the run's k-blocks
per split, calibrated by tests/test_mimi_plan_runs_cpu.py), the NaN-prefilled outputs fully written, a paused session's context bit for bit unchanged,
an executing session's committed context equal to the last P steps of its activated input (ELU where the layer has it; the
context is stored after the activation) within the hi / lo split's 2^-23 (2^-22 where fp32 expm1f made the value), and a
second launch of the second chunk identical bit for bit (the split-K reduction sums in split order).

The file ends by checking that every (layer, run, end) was executed, and prints each layer's largest need of the constant.
On one H100 80GB HBM3 (132 SMs, power limit 700 W) it ran all 226 cases in 27 s; the largest need was 61 of 111 (encoder.9,
96 unsplit k-blocks), and no case needed more than 0.61 of its run's constant (decoder.3 at 512 sessions).
"""
import ctypes as C
import time

import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import MimiConfig
from tests.util import TC_CONV, TC_CONVTR, cptr, mimi_plan_runs, mimi_tc_layers, tc_c, tc_op_shape, tc_ratios, tc_ref64

pytestmark = pytest.mark.gpu

LAYERS = mimi_tc_layers(MimiConfig())
_EXECUTED: set = set()
_NEED: dict = {}


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def env():
    lib = _lib.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return lib, sms, mimi_plan_runs(lib, sms)


def _elu32(x: torch.Tensor) -> torch.Tensor:
    return torch.where(x > 0, x, torch.expm1(x))


def _launch(lib, layer: dict, x, w, bias, prev, mask, B: int, T_in: int) -> torch.Tensor:
    tr = layer["kind"] == TC_CONVTR
    T_out = T_in * layer["stride"] if tr else T_in // layer["stride"]
    y = torch.full((B, layer["cout"], T_out), float("nan"), device="cuda")
    _lib.check(lib.b200_op_tc_conv1d(cptr(x), cptr(w), cptr(bias), cptr(prev), cptr(mask), cptr(y), B, layer["cin"], layer["cout"],
                                     T_in, layer["k"], layer["stride"], layer["dil"], int(layer["elu"]), int(tr), _st()))
    torch.cuda.synchronize()
    return y


def tc_conv_case(lib, layer: dict, B: int, T_in: int, g: torch.Generator, pause: int | None, what: str,
                 c: float) -> tuple[float, list]:
    """Two chunks of one layer through b200_op_tc_conv1d (the second with session ``pause`` paused) and every check of the
    module docstring, the outputs under the rule's constant c.  Returns (largest constant needed, failures)."""
    tr = layer["kind"] == TC_CONVTR
    cin, cout, k, st, dil = layer["cin"], layer["cout"], layer["k"], layer["stride"], layer["dil"]
    P = 1 if tr else (k - 1) * dil + 1 - st
    kind = TC_CONVTR if tr else TC_CONV
    w = ((torch.randn(cin, cout, k, generator=g, device="cuda") if tr else torch.randn(cout, cin, k, generator=g, device="cuda"))
         / (cin * k) ** 0.5)
    bias = 0.5 * torch.randn(cout, generator=g, device="cuda")
    ctx = torch.randn(B, cin, P, generator=g, device="cuda")
    prev = (_elu32(ctx) if layer["elu"] else ctx).contiguous() if P > 0 else None
    need, bad = 0.0, []
    for chunk in range(2):
        x = torch.randn(B, cin, T_in, generator=g, device="cuda")
        mask = torch.ones(B, dtype=torch.uint8, device="cuda")
        if chunk == 1 and pause is not None:
            mask[pause] = 0
        before = None if prev is None else prev.clone()
        y = _launch(lib, layer, x, w, bias, prev, mask, B, T_in)
        tag = f"{what} chunk {chunk}"
        if torch.isnan(y).any():
            bad.append(f"{tag}: {int(torch.isnan(y).sum())} outputs not written")
        want, scale = tc_ref64(kind, x, w, bias, before, stride=st, dil=dil, elu=layer["elu"])
        r = tc_ratios(y, want, scale, c)
        need = max(need, float(r.max()) * c)
        if float(r.max()) > 1:
            where = (r > 1).nonzero()[0].tolist()
            bad.append(f"{tag}: worst ratio {float(r.max()):.3g} (first failing output {where})")
        if prev is not None:
            a = x.double()
            act = torch.nn.functional.elu(a) if layer["elu"] else a
            ext = torch.cat([before.double(), act], dim=-1)[..., -P:]
            tol = 2.0 ** -23 * ext.abs()
            if layer["elu"]:
                made = torch.cat([torch.zeros_like(before, dtype=torch.bool), x < 0], dim=-1)[..., -P:]
                tol = torch.where(made, 2.0 ** -22 * ext.abs(), tol)
            ex = mask.bool()
            err = (prev.double() - ext).abs()
            if bool((err[ex] > tol[ex]).any()):
                bad.append(f"{tag}: committed context off its activated input by {float((err[ex] / tol[ex].clamp(min=1e-300)).max()):.3g} "
                           f"of the split's bound")
            if not bool(ex.all()) and not torch.equal(prev[~ex].view(torch.int32), before[~ex].view(torch.int32)):
                bad.append(f"{tag}: a paused session's context changed")
        if chunk == 1:
            again = None if before is None else before.clone()
            y2 = _launch(lib, layer, x, w, bias, again, mask, B, T_in)
            if not torch.equal(y2.view(torch.int32), y.view(torch.int32)) or (
                    again is not None and not torch.equal(again.view(torch.int32), prev.view(torch.int32))):
                bad.append(f"{tag}: a second launch differs")
    return need, bad


def _pause_row(B: int, bb: int) -> int:
    """The first session of the second session group, or the last session when there is one group."""
    return bb if bb < B else B - 1


@pytest.mark.parametrize("name", list(LAYERS))
def test_every_layer_at_both_ends_of_every_plan_run(env, name):
    lib, sms, table = env
    layer = LAYERS[name]
    shape = table["shapes"][name]
    T = shape[-1]
    assert tc_op_shape(layer, T) == shape[1:], (name, tc_op_shape(layer, T), shape)
    T_in = T if layer["kind"] == TC_CONVTR else T * layer["stride"]
    g = torch.Generator(device="cuda").manual_seed(len(name) * 1009 + T)
    t0 = time.time()
    failures = []
    for first, last, f in table["runs"][name]:
        tt, bb, ksplit, kbps = f[:4]
        for B in sorted({first, last}):
            what = f"{name} run {first}-{last} (tile {tt} x {bb}, {ksplit} x {kbps} over {shape[8]} k-blocks) B={B}"
            need, bad = tc_conv_case(lib, layer, B, T_in, g, _pause_row(B, bb), what, tc_c(kbps))
            print(f"\n{what}: constant {tc_c(kbps):.3g}, needed {need:.3g}", end="")
            _NEED[name] = max(_NEED.get(name, 0.0), need)
            failures += bad
            _EXECUTED.add((name, first, last, B))
    print(f"\n{name}: {len(table['runs'][name])} runs in {time.time() - t0:.1f} s, largest constant needed {_NEED[name]:.3g}")
    assert not failures, "\n".join(failures[:20])


def test_zz_every_run_end_was_executed(env, request):
    """Every run of every layer ran at its first and last session count.  It reads what the test above recorded, so it only
    judges a run of the whole file: under -k or a single test id it skips."""
    mine = [i for i in request.session.items if i.module is request.module]
    if len(mine) < len(LAYERS) + 1:
        pytest.skip("only part of this file was selected: coverage is judged on a run of the whole file")
    lib, sms, table = env
    want = {(n, a, b, B) for n, runs in table["runs"].items() for a, b, _ in runs for B in (a, b)}
    missing = sorted(want - _EXECUTED)
    print(f"\n{len(want)} (layer, run, end) cases at {sms} SMs, {len(want & _EXECUTED)} executed; largest constant needed per layer: "
          + ", ".join(f"{n} {v:.3g}" for n, v in _NEED.items()))
    assert not missing, missing[:20]
