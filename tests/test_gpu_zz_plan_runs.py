"""GPU: every plan the LM can take for its linears and for the fused depformer, at the first and last batch of each run.

The runs come from the library's own plan functions (tests/util.py linear_plan_runs / depformer_plan_runs) at this device's SM
count and the library's current GEMV limit, so a change of plan_linear or plan_depformer moves the tested batches with it.

Linears: every shape key of tests/golden/linear_plans.json, bf16 and int8 as the table lists them, through the entry point
that runs the LM's launches: b200_op_linear_sk with no force (b200_op_linear_sk_norm where the plan folds the RMSNorm into the
GEMV; above the GEMV limit the plan with the norm must equal the plan without it, which is what norm_linear launches after
rmsnorm_kernel), and b200_op_quant_pack_tiles / b200_op_quantize_rows / b200_op_linear_i8 for int8.  bf16 outputs are held to
the per-linear fp64 rule (tests/util.py linear_ratios, calibrated by tests/test_plan_runs_cpu.py), and >= 99 % of stored outputs
must equal bf16 of the fp64 product; int8 outputs, quantised rows and scales must equal oracle/quant.py bit for bit (the gated
epilogue: up to one bf16 ulp of silu).  Around every launch: the output sits between guard rows of NaN patterns that must come
back untouched, the residual input is unchanged, the in-place residual add (y == res, as the LM calls it) equals the
out-of-place one bit for bit, and a second launch repeats the first bit for bit (the split-K counters reset themselves).

Fused depformer: the 7b, 2b and ragged members of tests/test_gpu_zz_depformer_ref.py, default mode, at the first and last batch
of every fused run (batches that file already runs are listed as covered there), greedy, and sampled at the last batch of each
7B run; and the GEMV limit 4 at 3 and 4 sessions, where the plan takes the launch chain.  Its rule and checkpoints apply.

The file ends by checking that every run was executed or is covered (on a run of the whole file; a partial selection skips
that check).  On one H100 80GB HBM3 (132 SMs, power limit 700 W, GEMV limit 2) it runs 897 of the 908 (run, batch) pairs and
finds the other 11 covered, in about 75 s.  bf16 linears: every output within the rule, needing a slack constant of at most 4
of LINEAR_C = 32, >= 99.77 % of stored outputs equal to bf16(fp64); int8 linears bit-exact.  Depformer worst ratios (din,
layer-0 k / v, any k / v, logits): 7b 0.48, 0.44, 0.68, 0.58; 2b 0.48, 0.46, 0.63, 0.61; ragged 0.47, 0.43, 0.45, 0.24; no
unexcused token and no sampler mismatch.
"""
import ctypes as C
import json
import time
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from moshi_b200 import _lib
from oracle import quant
from tests.test_gpu_zz_depformer_ref import CASES, MEMBERS, _model, _run, _state_dict
from tests.util import (DEPFORMER_PHASES, DEPFORMER_PLAN_FIELDS, GATE, LINEAR_KERNELS, RESADD, STORE, _bf, bf_next_down,
                        bf_next_up, cptr, depformer_plan, depformer_plan_runs, linear_c_needed, linear_plan, linear_plan_runs,
                        linear_ratios, linear_ref64, linear_rows)

pytestmark = pytest.mark.gpu

TABLE = json.loads((Path(__file__).resolve().parent / "golden" / "linear_plans.json").read_text())
KEYS = list(TABLE["plans"])
NAMES = {}
for _n, _v in TABLE["shapes"].items():
    for _i8 in (0, 1):
        NAMES.setdefault(",".join(map(str, _v + [_i8])), _n + (".int8" if _i8 else ".bf16"))
GUARD = 256                  # rows of NaN patterns on each side of an output
FUSED, AUTO = 2, _lib.B200_DEPFORMER_AUTO
DEP_MEMBERS = ("7b", "2b", "ragged")

# what ran: ("linear", key, M) and ("dep", member, B); what test_gpu_zz_depformer_ref.py runs: ("dep", member, B)
_EXECUTED: set = set()
_COVERED: set = set()
_WORST: dict = {"c": 0.0}


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def env():
    lib = _lib.lib()
    gemv = lib.b200_op_set_gemv_max_rows(2)
    lib.b200_op_set_gemv_max_rows(gemv)
    return lib, torch.cuda.get_device_properties(0).multi_processor_count, gemv


def _guarded(M: int, cols: int) -> tuple[torch.Tensor, torch.Tensor]:
    """(whole buffer as int16, the [M, cols] bf16 view between GUARD rows of NaN patterns on each side)."""
    n = (2 * GUARD + M) * cols
    buf = (torch.arange(n, device="cuda", dtype=torch.int32) % 63 + 0x7F81).to(torch.int16)
    return buf, buf[GUARD * cols:(GUARD + M) * cols].view(torch.bfloat16).view(M, cols)


def _guards_intact(buf: torch.Tensor, M: int, cols: int) -> bool:
    n = (2 * GUARD + M) * cols
    pat = (torch.arange(n, device="cuda", dtype=torch.int32) % 63 + 0x7F81).to(torch.int16)
    lo, hi = GUARD * cols, (GUARD + M) * cols
    return torch.equal(buf[:lo], pat[:lo]) and torch.equal(buf[hi:], pat[hi:])


def _launch_checked(call, M: int, cols: int, res: torch.Tensor | None, what: str) -> torch.Tensor:
    """Runs call(y, res) into a guarded output twice and in place (residual add): returns y after every edge check."""
    res0 = None if res is None else res.clone()
    outs = []
    for _ in range(2):
        buf, y = _guarded(M, cols)
        _lib.check(call(y, res))
        torch.cuda.synchronize()
        assert _guards_intact(buf, M, cols), f"{what}: a guard row next to the output changed"
        outs.append(y)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), f"{what}: a second launch differs"
    if res is not None:
        assert torch.equal(res, res0), f"{what}: the residual input changed"
        buf, y = _guarded(M, cols)
        y.copy_(res)
        _lib.check(call(y, y))
        torch.cuda.synchronize()
        assert _guards_intact(buf, M, cols), f"{what}: a guard row next to the in-place output changed"
        assert torch.equal(y.view(torch.int16), outs[0].view(torch.int16)), f"{what}: in place differs from out of place"
    return outs[0]


def _describe(launches: list) -> str:
    return "+".join(f"{LINEAR_KERNELS[b[0]]}[{b[2]}]" for b in launches)


def _bf16_case(lib, key, M, w, wt, alpha, sms, gemv, g):
    N, K, epi, H, norm, _ = map(int, key.split(","))
    cols = H if epi == GATE else N
    x = linear_rows(M, K, g, "cuda")
    res = torch.randn(M, cols, generator=g, device="cuda").bfloat16() if epi == RESADD else None
    folded, launches = linear_plan(lib, M, N, K, epi, H, norm, 0, sms, gemv)
    if norm and not folded:
        # norm_linear: rmsnorm_kernel, then the launches of the plan without a norm
        assert linear_plan(lib, M, N, K, epi, H, 0, 0, sms, gemv) == (0, launches), (key, M)
    if folded:
        call = lambda y, r: lib.b200_op_linear_sk_norm(cptr(x), cptr(alpha), cptr(wt), cptr(y), cptr(r), M, N, K, epi, H, _st())
    else:
        call = lambda y, r: lib.b200_op_linear_sk(cptr(x), cptr(wt), cptr(y), cptr(r), M, N, K, epi, H, 0, 0, 0, _st())
    what = f"{NAMES[key]} M={M}"
    y = _launch_checked(call, M, cols, res, what)
    ref = linear_ref64(x, w, epi, H, res, alpha=alpha if folded else None)
    worst = float(linear_ratios(y, ref).max())
    c = linear_c_needed(y, ref)
    _WORST["c"] = max(_WORST["c"], c)
    exact = float((y.double() == _bf(ref["acc"])).double().mean()) if epi == STORE else 1.0
    bad = []
    if worst > 1:
        bad.append(f"{what}: worst ratio {worst:.3g}")
    if exact < 0.99:
        bad.append(f"{what}: only {exact:.4f} of the outputs equal bf16 of the fp64 product")
    # (a faithful rounding on the far side of the reference scores exactly 1: the slack it needs is the informative number)
    return launches, f"{'within' if worst <= 1 else 'outside'} the rule, slack constant needed {c:g}, {exact:.4f} exact", bad


def _int8_case(lib, key, M, w, wt, sw, sms, gemv, g):
    N, K, epi, H, norm, _ = map(int, key.split(","))
    cols = H if epi == GATE else N
    x = linear_rows(M, K, g, "cuda")
    res = torch.randn(M, cols, generator=g, device="cuda").bfloat16() if epi == RESADD else None
    _, launches = linear_plan(lib, M, N, K, epi, H, norm, 1, sms, gemv)
    xq = torch.empty(M, K, dtype=torch.int8, device="cuda")
    sa = torch.empty(M, dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_op_quantize_rows(cptr(x), cptr(xq), cptr(sa), M, K, _st()))
    call = lambda y, r: lib.b200_op_linear_i8(cptr(xq), cptr(sa), cptr(wt), cptr(sw), cptr(y), cptr(r), M, N, K, epi, H, _st())
    what = f"{NAMES[key]} M={M}"
    y = _launch_checked(call, M, cols, res, what)
    qx, sa_o = quant.quantize_rows(x)
    qw, sw_o = quant.quantize_weight(w)
    bad = []
    if not (torch.equal(xq, qx) and torch.equal(sa, sa_o)):
        bad.append(f"{what}: quantised rows differ from oracle/quant.py")
    h = quant.qproduct_f32(qx, sa_o, qw, sw_o)
    if epi == STORE:
        ok = y.view(torch.int16) == h.bfloat16().view(torch.int16)
    elif epi == RESADD:
        ok = y.view(torch.int16) == (res.float() + h.bfloat16().float()).bfloat16().view(torch.int16)
    else:
        hb = h.bfloat16()
        s = F.silu(hb[:, :H].float()).bfloat16().double()
        u = hb[:, H:].double()
        yd = y.double()
        # one bf16 ulp of silu (expf on the device): y must be the product of silu's bf16 or one of its neighbours
        ok = torch.zeros_like(yd, dtype=torch.bool)
        for sv in (s, bf_next_up(s), bf_next_down(s)):
            ok |= yd == _bf(sv * u)
    mism = int((~ok).sum())
    if mism:
        bad.append(f"{what}: {mism} outputs differ from oracle/quant.py")
    return launches, f"{mism} outputs off the oracle", bad


@pytest.mark.parametrize("key", KEYS, ids=[NAMES[k] for k in KEYS])
def test_every_linear_plan_run(env, key):
    lib, sms, gemv = env
    N, K, epi, H, norm, int8 = map(int, key.split(","))
    t0 = time.time()
    g = torch.Generator(device="cuda").manual_seed(N * 7 + K + epi + int8)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).bfloat16()
    alpha = (torch.rand(K, generator=g, device="cuda") + 0.5).bfloat16() if norm else None
    if int8:
        wt = torch.empty(lib.b200_op_packed_bytes_i8(N, K, epi, H), dtype=torch.uint8, device="cuda")
        sw = torch.empty(N, dtype=torch.float32, device="cuda")
        _lib.check(lib.b200_op_quant_pack_tiles(cptr(w), cptr(wt), cptr(sw), N, K, epi, H, _st()))
        torch.cuda.synchronize()
        assert torch.equal(sw, quant.quantize_weight(w)[1]), f"{NAMES[key]}: weight scales differ from oracle/quant.py"
    else:
        wt = torch.empty(lib.b200_op_packed_bytes(N, K, epi, H), dtype=torch.uint8, device="cuda")
        _lib.check(lib.b200_op_pack_tiles(cptr(w), cptr(wt), N, K, epi, H, _st()))
    failures = []
    runs = linear_plan_runs(lib, N, K, epi, H, norm, int8, sms, gemv)
    for first, last, _ in runs:
        for M in sorted({first, last}):
            if int8:
                launches, line, bad = _int8_case(lib, key, M, w, wt, sw, sms, gemv, g)
            else:
                launches, line, bad = _bf16_case(lib, key, M, w, wt, alpha, sms, gemv, g)
            print(f"\n{NAMES[key]} run {first}-{last} M={M}: {_describe(launches)}: {line}", end="")
            failures += bad
            _EXECUTED.add(("linear", key, M))
    print(f"\n{NAMES[key]}: {len(runs)} runs in {time.time() - t0:.1f} s")
    assert not failures, "\n".join(failures[:20])


def _dep_batches(member: str, runs: list) -> list[tuple[int, bool, tuple]]:
    """(B, sampled, run) of the fused runs not already run by test_gpu_zz_depformer_ref.py; records what it covers."""
    done = {B for c in CASES if c[0] == member and c[1] == "fused" for B in c[3]}
    sampled = {B for c in CASES if c[0] == member and c[1] == "fused" for B in c[4]}
    out = []
    for first, last, p in runs:
        if p[0] != FUSED:
            continue
        for B in sorted({first, last}):
            smp = member == "7b" and B == last and B not in sampled
            if B in done:
                _COVERED.add(("dep", member, B))
                print(f"\n{member} run {first}-{last} B={B}: covered by test_gpu_zz_depformer_ref.py", end="")
            if B not in done or smp:
                out.append((B, smp, (first, last)))
    return out


def _splits(p: list) -> str:
    return " ".join(f"{ph} {p[DEPFORMER_PLAN_FIELDS.index(ph + '.S')]}" for ph in DEPFORMER_PHASES)


@pytest.mark.parametrize("member", DEP_MEMBERS)
def test_every_fused_depformer_plan_run(env, member):
    lib, sms, gemv = env
    cfg = MEMBERS[member]
    geom = (cfg.dep_q, cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_ffn_hidden, cfg.card)
    runs = depformer_plan_runs(lib, geom, 0, 0, AUTO, sms, gemv)
    t0 = time.time()
    sd = _state_dict(member)
    lm = _model(cfg, sd, AUTO)
    g = torch.Generator().manual_seed(977 + len(member))
    min_launches = cfg.dep_q * cfg.depformer_num_layers * 5      # the launch chain: one launch per linear or attention at least
    cases = [(B, smp, run, gemv) for B, smp, run in _dep_batches(member, runs)] + [(B, False, None, 4) for B in (3, 4)]
    failures = []
    try:
        for B, smp, run, limit in cases:
            p = depformer_plan(lib, geom, B, 0, 0, AUTO, sms, limit)
            for sampling in ((False, True) if smp else (False,)):
                if sampling is False and run is not None and ("dep", member, B) in _COVERED:
                    continue                      # run greedy there; only the sampled case is new
                before = lib.b200_op_set_gemv_max_rows(limit)    # the plan is made at streaming_begin
                try:
                    res = _run(lm, member, sd, B, sampling, g)
                finally:
                    lib.b200_op_set_gemv_max_rows(before)
                w = res["worst"]
                kv = " ".join(f"{w[f'k{l}']:.3f}/{w[f'v{l}']:.3f}" for l in range(cfg.depformer_num_layers))
                where = f"run {run[0]}-{run[1]}" if run else f"GEMV limit {limit}"
                path = "fused" if p[0] == FUSED else "chain"
                print(f"\n{member} {where} B={B} {'sampled' if sampling else 'greedy'} ({path}; splits {_splits(p)}; partial "
                      f"floats {p[1]}; launches per step {res['launches']}): worst ratio din {w['din']:.3f}, k/v per layer {kv}, "
                      f"logits {w['logits']:.3f}; tokens differing {res['differ']}/{res['decisions']} "
                      f"({res['unexcused']} unexcused), sampler mismatches {res['sampler']}", end="")
                tag = f"{member} {where} B={B} {'sampled' if sampling else 'greedy'}"
                if (max(res["launches"]) >= min_launches) == (p[0] == FUSED):
                    failures.append(f"{tag}: {res['launches']} launches per step on the {path} path")
                if res["first"] is not None:
                    failures.append(f"{tag}: first failing {res['first']}")
                if res["unexcused"] or res["sampler"]:
                    failures.append(f"{tag}: {res['unexcused']} unexcused token differences, {res['sampler']} sampler mismatches")
                if run is not None:
                    _EXECUTED.add(("dep", member, B))
    finally:
        del lm
        torch.cuda.empty_cache()
    print(f"\n{member}: {len(cases)} batches in {time.time() - t0:.1f} s")
    assert not failures, "\n".join(failures)


def test_zz_every_run_was_executed_or_covered(env, request):
    """Every run of every linear shape and every fused-depformer run of the 7b, 2b and ragged members, at its first and last
    batch, ran in this file or in test_gpu_zz_depformer_ref.py.  It reads what the tests above recorded, so it only judges a
    run of the whole file: under -k or a single test id it skips."""
    mine = [i for i in request.session.items if i.module is request.module]
    if len(mine) < len(KEYS) + len(DEP_MEMBERS) + 1:
        pytest.skip("only part of this file was selected: coverage is judged on a run of the whole file")
    lib, sms, gemv = env
    want = set()
    for key in KEYS:
        N, K, epi, H, norm, int8 = map(int, key.split(","))
        for first, last, _ in linear_plan_runs(lib, N, K, epi, H, norm, int8, sms, gemv):
            want |= {("linear", key, first), ("linear", key, last)}
    for member in DEP_MEMBERS:
        cfg = MEMBERS[member]
        geom = (cfg.dep_q, cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_ffn_hidden, cfg.card)
        for first, last, p in depformer_plan_runs(lib, geom, 0, 0, AUTO, sms, gemv):
            if p[0] == FUSED:
                want |= {("dep", member, first), ("dep", member, last)}
    missing = sorted(want - _EXECUTED - _COVERED)
    print(f"\n{len(want)} (plan run, batch) pairs at {sms} SMs and GEMV limit {gemv}: {len(want & _EXECUTED)} executed here, "
          f"{len(want & _COVERED - _EXECUTED)} covered by test_gpu_zz_depformer_ref.py; bf16 linears: largest slack constant "
          f"needed {_WORST['c']:g}")
    assert not missing, missing[:20]
