"""CPU: the plan runs the GPU tests derive from the library, and the per-linear fp64 rule they apply.

tests/test_gpu_zz_plan_runs.py runs every linear and every fused-depformer plan at the first and last batch of each run, the
runs being derived from b200_op_linear_plan / b200_op_depformer_plan at the device's SM count.  Here, at 132 SMs and the default
GEMV limit, that derivation must reproduce the run boundaries of tests/golden/linear_plans.json and depformer_plans.json.

The rule of one linear (tests/util.py linear_ratios) must accept fp32 emulations of the linear in several summation orders (per
k-block, per K-split, in reverse) and reject each of these kernel bugs on shapes with a ragged K tail: a lost k-block, a k-block
counted twice, a lost tail of 8 columns, one split's partial added twice, the rows of a second row block read one row late (a
wrong m0) and the weights of the neighbouring 128-row tile.  The slack constant is pinned below: loosening it fails this file.
"""
import json
import math
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from tests.util import (GATE, LINEAR_C, NORM_BAND, RESADD, STORE, _bf, depformer_plan_runs, linear_c_needed, linear_plan_runs,
                        linear_ratios, linear_ref64, linear_rows)

GOLDEN = Path(__file__).resolve().parent / "golden"
BLOCK_K = 64


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    from moshi_b200.build import build
    build()
    return _lib.lib()


def test_linear_plan_runs_reproduce_the_golden_table(lib):
    t = json.loads((GOLDEN / "linear_plans.json").read_text())
    for k, runs in t["plans"].items():
        N, K, epi, gate_rows, norm, int8 = map(int, k.split(","))
        got = linear_plan_runs(lib, N, K, epi, gate_rows, norm, int8, t["sms"], t["gemv_max_rows"], t["max_m"])
        assert [(a, b) for a, b, _ in got] == [(r[0], r[1]) for r in runs], k
        assert [blocks for _, _, blocks in got] == [r[3] for r in runs], k


def test_depformer_plan_runs_reproduce_the_golden_table(lib):
    t = json.loads((GOLDEN / "depformer_plans.json").read_text())
    for k, runs in t["plans"].items():
        v = list(map(int, k.split(",")))
        geom, (cfg, int8, mode, gemv) = v[:5], v[5:]
        got = depformer_plan_runs(lib, geom, cfg, int8, mode, t["sms"], gemv, t["max_b"])
        assert [(a, b) for a, b, _ in got] == [(r[0], r[1]) for r in runs], k
        assert [p for _, _, p in got] == [r[2] for r in runs], k


def test_the_slack_constants_are_pinned():
    """LINEAR_C: 32 fp32 roundings of sum_k |x_k w_k|, the most the rule grants an fp32 product summed in another order (the
    kernels need at most 4 on an H100; every mutant below needs 2^16 or more).  NORM_BAND: how close to a bf16 midpoint an
    fp32 RMSNorm output may round the other way."""
    assert LINEAR_C <= 32.0
    assert NORM_BAND <= 2.0 ** -16


# ---- fp32 emulations of one linear ------------------------------------------------------------------------------------------
def _blocks(K: int) -> list[tuple[int, int]]:
    return [(k, min(k + BLOCK_K, K)) for k in range(0, K, BLOCK_K)]


def _splits(n: int, S: int) -> list[list[int]]:
    """k-block indices of S K-splits, as the kernels cut them: ceil(n / S) per split, the last one ragged."""
    per = -(-n // S)
    return [list(range(s, min(s + per, n))) for s in range(0, n, per)]


def _acc32(x: torch.Tensor, w: torch.Tensor, order: str = "forward", S: int = 3, mutant: str | None = None) -> torch.Tensor:
    """fp32 x . w^T summed per 64-column k-block (each block an fp32 product), the blocks added in `order`: forward, reverse, or
    per split (blocks summed within each of S splits, the split partials added in split order); `mutant` a kernel bug."""
    K = x.shape[1]
    blocks = _blocks(K)
    if mutant == "lost ragged tail of 8 columns":
        blocks[-1] = (blocks[-1][0], K - 8)
    part = [x[:, a:b].float() @ w[:, a:b].float().t() for a, b in blocks]
    mid = len(blocks) // 2
    idx = list(range(len(blocks)))
    if mutant == "lost k-block":
        idx.remove(mid)
    elif mutant == "k-block counted twice":
        idx.insert(mid, mid)
    if order == "reverse":
        idx = idx[::-1]
    groups = _splits(len(blocks), S) if order == "split" or mutant == "split partial added twice" else [idx]
    if mutant == "split partial added twice":
        groups.insert(1, groups[1])
    total = torch.zeros_like(part[0])
    for grp in groups:
        p = torch.zeros_like(part[0])
        for j in grp:
            p = p + part[j]
        total = total + p
    return total


def _epilogue(acc: torch.Tensor, epi: int, H: int, res: torch.Tensor | None) -> torch.Tensor:
    """The kernels' epilogues in fp32 with their bf16 cast points."""
    if epi == STORE:
        return acc.bfloat16()
    if epi == RESADD:
        return (res.float() + acc.bfloat16().float()).bfloat16()
    g, u = acc[:, :H].bfloat16().float(), acc[:, H:].bfloat16().float()
    return (F.silu(g).bfloat16().float() * u).bfloat16()


# (M, N, K, epi, rows per launch): K tails of 40, 8 and 40 columns; N with a partial 128-row tile; more rows than one launch
SHAPES = [(40, 384, 1000, STORE, 128), (200, 384, 2824, RESADD, 128), (70, 600, 1000, GATE, 64), (3, 4096, 4104, STORE, 128),
          (160, 1000, 2824, STORE, 128)]
ORDERS = ["forward", "split", "reverse"]
MUTANTS = ["lost k-block", "k-block counted twice", "lost ragged tail of 8 columns", "split partial added twice",
           "second row block one row late", "neighbouring weight tile"]


def _case(M, N, K, epi, seed=0):
    g = torch.Generator().manual_seed(seed + M + N + K)
    x = linear_rows(M, K, g)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    H = N // 2 if epi == GATE else 0
    res = torch.randn(M, N, generator=g).bfloat16() if epi == RESADD else None
    return x, w, H, res


@pytest.mark.parametrize("M,N,K,epi,block", SHAPES)
def test_rule_accepts_fp32_in_every_order_and_rejects_every_mutant(M, N, K, epi, block):
    x, w, H, res = _case(M, N, K, epi)
    ref = linear_ref64(x, w, epi, H, res)
    for order in ORDERS:
        y = _epilogue(_acc32(x, w, order), epi, H, res)
        r = linear_ratios(y, ref)
        print(f"{M}x{N}x{K} epi={epi} {order}: slack constant needed {linear_c_needed(y, ref):g}")
        assert float(r.max()) <= 1, order
        if epi == STORE:
            assert float((y.double() == _bf(ref["acc"])).double().mean()) >= 0.99, order
    good = _epilogue(_acc32(x, w), epi, H, res)
    for name in MUTANTS:
        xm, wm = x, w
        if name == "second row block one row late":
            if M <= block:
                continue
            xm = x.clone()
            xm[block:M - 1] = x[block + 1:M]
            xm[M - 1] = 0
        elif name == "neighbouring weight tile":
            wm = w.clone()
            for base in ((0, H) if epi == GATE else (0,)):
                wm[base:base + 128] = w[base + 128:base + 256]
        y = _epilogue(_acc32(xm, wm, mutant=name), epi, H, res)
        r = linear_ratios(y, ref).max(-1).values
        changed = (y != good).any(-1)
        if epi == RESADD:
            # the update of the row scaled by 1e-3 sits below the rounding of the residual: no rule can see a bug in it there
            changed[0] = False
        admitted = [m for m in changed.nonzero().flatten().tolist() if float(r[m]) <= 1]
        # the smallest slack constant that would admit the mutant
        c = LINEAR_C
        while c < 2.0 ** 40 and float(linear_ratios(y, ref, c).max()) > 1:
            c *= 2
        print(f"{M}x{N}x{K} epi={epi} {name}: {int(changed.sum())} rows changed, {len(admitted)} admitted, "
              f"worst ratio {float(r.max()):.3g}, admitted from LINEAR_C = {c:.3g}")
        assert int(changed.sum()) > 0, name
        assert not admitted, (name, admitted[:8])
        assert c >= 64 * LINEAR_C, (name, c)


@pytest.mark.parametrize("M,K", [(1, 4096), (2, 2560), (2, 1024)])
@pytest.mark.parametrize("epi", [STORE, RESADD, GATE])
def test_rule_accepts_an_fp32_rmsnorm_in_front(M, K, epi):
    """The RMSNorm folded into the GEMV (fp32 sum of squares, rsqrt, x * (alpha * r), bf16) then the linear: accepted against
    linear_ref64 with alpha; the same linear over the unnormalised rows is not."""
    g = torch.Generator().manual_seed(M * K + epi)
    x = linear_rows(M, K, g) * 3
    alpha = (torch.rand(K, generator=g) + 0.5).bfloat16()
    N = 768
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    H = N // 2 if epi == GATE else 0
    res = torch.randn(M, N, generator=g).bfloat16() if epi == RESADD else None
    xf = x.float()
    r = torch.rsqrt(1e-8 + (xf * xf).sum(-1, keepdim=True) / K)
    xn = (xf * (alpha.float() * r)).bfloat16()
    ref = linear_ref64(x, w, epi, H, res, alpha=alpha)
    for order in ORDERS:
        y = _epilogue(_acc32(xn, w, order), epi, H, res)
        assert float(linear_ratios(y, ref).max()) <= 1, order
    y = _epilogue(_acc32(x, w), epi, H, res)
    assert math.isinf(float(linear_ratios(y, ref).max())) or float(linear_ratios(y, ref).max()) > 1
