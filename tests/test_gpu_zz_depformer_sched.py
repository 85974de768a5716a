"""GPU: depformer weight-sharing schedules and low-rank depformer embeddings (lm.py:125-127, 172-196; transformer.py:291-316,
399-401; lm_utils.py:80-124).

* The reference-recorded fixture tests/golden/lm_tiny_sched.* (tools/gen_golden_sched.py: schedule [0, 1, 2, 2, 2, 3, 3, 3],
  rank 32): the handle is teacher-synchronised on the oracle, text logits within LOGIT_ATOL, sampled tokens bit-exact given
  the handle's own logits, and rows on the fixture's greedy trajectory reproduce it up to provable bf16 near-ties.
* Every depformer checkpoint of a frame (din of every weight set, k / v of every layer and sub-step, logits) against
  depformer_ref64 (tests/util.py) under its rules, on geometries whose weight sets all hold distinct random weights, so that a
  wrong set index or a wrong din column fails: the 7B depformer with a schedule and rank 128, a 16-sub-step member with
  schedule [0..7, 8 x 8], and a cross-attention member (the TTS models' LM) with a schedule and rank 64.  Batches 1 and 2 (GEMV chain), 3, 40 and 256 (persistent kernel), both paths forced, classifier-free
  guidance (chain) and int8 linears, under which every expanded table row equals oracle/quant.py's QLinear on that row.
* A schedule keeps each shared set resident once: the device memory a scheduled model takes is smaller by dep_q - n_sets weight
  sets.  A scheduled, low-rank handle continues bit for bit after a session export / import and a state round trip.
"""
import dataclasses
import json

import pytest
import torch
from safetensors.torch import load_file

from moshi_b200 import _lib
from moshi_b200.config import LMConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict
from oracle import scenarios
from oracle.lm import LMOracle, sample_token
from tests.depformer_sched import sched_spec
from tests.util import (cfg_guide64, dep_checkpoints, dep_row_ratios, dep_row_scaled, depformer_ref64,
                        exact_row_ratios, greedy_unexcused, sample_is_stable, sampler_mismatches)

pytestmark = pytest.mark.gpu

AUTO, CHAIN, FUSED = _lib.B200_DEPFORMER_AUTO, _lib.B200_DEPFORMER_CHAIN, _lib.B200_DEPFORMER_FUSED
LOGIT_ATOL = 0.05
SMP = dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25)

MEMBERS = {
    # one temporal layer of the 7B shape in front of the full 7B depformer, 4 weight sets over 8 sub-steps, rank-128 tables
    "7b": LMConfig(num_layers=1, context=16, depformer_weights_per_step_schedule=[0, 1, 2, 2, 2, 3, 3, 3],
                   depformer_low_rank_embeddings=128),
    # 16 sub-steps over 9 weight sets, full-rank tables
    "q16": LMConfig(dim=1024, num_heads=8, num_layers=1, context=16, text_card=4000, n_q=32, dep_q=16, depformer_context=16,
                    depformer_num_layers=2, delays=[0, 0] + [2] * 15 + [0] + [2] * 15,
                    depformer_weights_per_step_schedule=list(range(8)) + [8] * 8),
    # a cross-attention member (the TTS models' LM, tests/test_gpu_zz_cross_ref.py's small geometry): 4 sub-steps over 3 sets,
    # rank-64 tables, every temporal layer attending to a per-session condition memory
    "cross": LMConfig.from_dict({"dim": 2048, "num_heads": 16, "num_layers": 1, "context": 16, "text_card": 8000, "n_q": 8,
                                 "dep_q": 4, "delays": [0] + [1] * 8, "depformer_num_layers": 2, "cross_attention": True,
                                 "conditioners": {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 512}}},
                                 "fuser": {"cross": ["speaker_wavs"]}, "depformer_weights_per_step_schedule": [0, 1, 1, 2],
                                 "depformer_low_rank_embeddings": 64}),
}
# (member, name, depformer mode, batches, of which also sampled, options)
CASES = [
    ("7b", "auto", AUTO, (1, 2, 3, 40, 256), (2, 40)),
    ("7b", "chain", CHAIN, (3, 40), (40,)),
    ("7b", "fused-forced", FUSED, (1,), (1,)),
    ("q16", "auto", AUTO, (1, 3, 40), (40,)),
    ("q16", "chain", CHAIN, (40,), ()),
    ("cross", "auto", AUTO, (1, 3, 40), (3,)),
    ("cross", "chain", CHAIN, (40,), ()),
]
CASES_OPT = [
    ("7b", "cfg3", (2, 40), (40,), dict(cfg=3.0)),
    ("7b", "int8", (1, 3, 40), (40,), dict(int8=True)),
]
FRAMES = 2


def _model(cfg, sd, mode=AUTO):
    from moshi_b200.models import LMModel
    lm = LMModel(cfg, sd, device="cuda")
    _lib.check(_lib.lib().b200_lm_set_depformer(lm._h, mode))
    return lm


def _conditions(lm, B: int, g: torch.Generator):
    """Condition tensors of B random voices [1, 20, 512] (each session its own condition memory)."""
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(torch.randn(1, 20, 512, generator=g))})
             for _ in range(B)]
    return lm.condition_provider(lm.condition_provider.prepare(attrs))


def _tables(gen, cfg) -> list[torch.Tensor]:
    return [gen.read_buffer(f"depformer.tables.{k}", torch.bfloat16, ((cfg.text_card if k == 0 else cfg.card) + 1,
                                                                      cfg.depformer_dim)) for k in range(cfg.dep_q)]


def _table_faults(sd: dict, cfg, tables: list[torch.Tensor], int8: bool) -> list[str]:
    """Every expanded row against its definition.  bf16: within half a bf16 ulp of the exact product plus the error bound of
    r fp32 sums (r 2^-24 sum_i |e_i w_i|, which matters where the terms cancel); int8: oracle/quant.py's QLinear of the row,
    bit for bit."""
    from oracle.quant import qlinear
    bad = []
    for k, got in enumerate(tables):
        name = "depformer_text_emb" if k == 0 else f"depformer_emb.{k - 1}"
        e, low = sd[name + ".weight"], sd.get(name + ".low_rank.weight")
        if low is None:
            ok = bool(torch.equal(got, e.to(got.device)))
        elif int8:
            ok = bool(torch.equal(got.cpu(), qlinear(e.cpu(), low.cpu())))
        else:
            want = e.double() @ low.double().T
            g = got.double().to(want.device)
            half_ulp = torch.ldexp(torch.ones_like(want), torch.frexp(want)[1] - 9)
            bound = half_ulp + low.shape[1] * 2.0 ** -24 * (e.double().abs() @ low.double().abs().T)
            ok = bool(((g - want).abs() <= bound).all())
        if not ok:
            bad.append(f"table {k}")
    return bad


def _weight_mutant(cfg, tables):
    """depformer_ref64 reads weights by sub-step: map them to the schedule's sets, and read the step's tables as expanded."""
    sched = cfg.depformer_weights_per_step_schedule or list(range(cfg.dep_q))

    def weight(name, k, layer, fetch):
        if name == "emb":
            return tables[k]
        if name in ("din", "in", "out", "lin_in", "lin_out"):
            return fetch(name, sched[k], layer)
        return fetch(name, k, layer)
    return dict(weight=weight)


@torch.no_grad()
def _run(lm, cfg, sd, B, sampling, g, opt) -> dict:
    from moshi_b200.models import LMGen
    coef = opt.get("cfg", 1.0)
    guided, int8 = coef != 1.0, bool(opt.get("int8"))
    ct = _conditions(lm, B, g) if cfg.cross_attention else None
    gen = LMGen(lm, use_sampling=sampling, cfg_coef=coef, cfg_is_no_text=guided, condition_tensors=ct, **SMP)
    Q, dd, H, L, card = cfg.dep_q, cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_num_layers, cfg.card
    sched = cfg.depformer_weights_per_step_schedule or list(range(Q))
    n_sets = cfg.depformer_n_sets
    kt, ka = min(SMP["top_k_text"], cfg.text_card), min(SMP["top_k"], card)
    res = dict(worst={}, first=None, sampler=0, unexcused=0, decisions=0, differ=0, tables=[])
    with gen.streaming(B):
        MB = gen._model_batch
        tables = _tables(gen, cfg)
        res["tables"] = _table_faults(sd, cfg, tables, int8)
        mutant = _weight_mutant(cfg, tables)
        for frame in range(FRAMES):
            codes = torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g).cuda()
            noise = torch.empty(B, kt + Q * ka).exponential_(1, generator=g).cuda() if sampling else None
            gen.step(codes, noise=noise)
            tout = gen.read_buffer("transformer_out", torch.bfloat16, (MB, cfg.dim))
            text = gen.read_buffer("text_token", torch.int64, (B,))
            toks = gen.read_buffer("audio_tokens", torch.int64, (Q, B))
            din_sets = gen.read_buffer("dep_in", torch.bfloat16, (MB, n_sets, dd))
            got = dict(din=din_sets[:, sched],
                       k=[gen.read_buffer(f"depformer.layers.{l}.k", torch.bfloat16, (MB, H, Q, 64)) for l in range(L)],
                       v=[gen.read_buffer(f"depformer.layers.{l}.v", torch.bfloat16, (MB, H, Q, 64)) for l in range(L)],
                       logits=gen.read_buffer("model_dep_logits", torch.bfloat16, (Q, MB, card)))
            rep = 2 if guided else 1
            want = depformer_ref64(sd, cfg, tout, text.repeat(rep), toks.repeat(1, rep), mutant=mutant, quantize=int8,
                                   din=got["din"])
            for kind, k, layer, gk, wk in dep_checkpoints(got, want):
                r = exact_row_ratios(gk, wk) if int8 and kind == "din" else dep_row_ratios(gk, wk, kind, layer, int8)
                key = kind if layer is None else f"{kind}{layer}"
                res["worst"][key] = max(res["worst"].get(key, 0.0), float(r.max()))
                if res["first"] is None and bool((r > 1).any()):
                    res["first"] = f"frame {frame} sub-step {k} layer {layer} {kind}: worst ratio {float(r.max()):.3g}"
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (Q, B, card))
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card))
            res["sampler"] += sampler_mismatches(tl, text, sampling, SMP["temp_text"], SMP["top_k_text"],
                                                 None if noise is None else noise[:, :kt])
            for k in range(Q):
                nk = None if noise is None else noise[:, kt + k * ka:kt + (k + 1) * ka]
                res["sampler"] += sampler_mismatches(dl[k], toks[k], sampling, SMP["temp"], SMP["top_k"], nk)
                wl = want["logits"][k]
                ref_lg = (cfg_guide64(wl, B, coef) if guided else wl.bfloat16()).float()
                ref_tok = sample_token(ref_lg, sampling, SMP["temp"], SMP["top_k"], nk, tie_break="index")
                res["decisions"] += B
                for b in (ref_tok != toks[k]).nonzero().flatten().tolist():
                    res["differ"] += 1
                    tol = float((dl[k][b].float() - ref_lg[b]).abs().max()) + 1e-6
                    if sampling:
                        res["unexcused"] += int(sample_is_stable(ref_lg[b:b + 1], SMP["temp"], SMP["top_k"], nk[b:b + 1], tol)[0])
                    else:
                        res["unexcused"] += greedy_unexcused(toks[k][b:b + 1], ref_tok[b:b + 1], ref_lg[b:b + 1].cpu(), tol)[1]
    return res


def _check(lm, cfg, sd, name, batches, sampled, opt, seed) -> list[str]:
    g = torch.Generator().manual_seed(seed)
    failures = []
    for B in batches:
        for sampling in (False, True) if B in sampled else (False,):
            res = _run(lm, cfg, sd, B, sampling, g, opt)
            w = res["worst"]
            mode = "sampled" if sampling else "greedy"
            print(f"\n{name} B={B} {mode}: worst ratios " + " ".join(f"{k} {v:.3f}" for k, v in w.items()) +
                  f"; tokens differing from the reference {res['differ']}/{res['decisions']} ({res['unexcused']} unexcused), "
                  f"sampler mismatches {res['sampler']}")
            if res["tables"]:
                failures.append(f"{name} B={B}: expanded tables differ from their definition: {res['tables']}")
            if res["first"] is not None:
                failures.append(f"{name} B={B} {mode}: first failing {res['first']}")
            if res["unexcused"] or res["sampler"]:
                failures.append(f"{name} B={B} {mode}: {res['unexcused']} unexcused, {res['sampler']} sampler mismatches")
    return failures


@pytest.mark.parametrize("member,name,mode,batches,sampled", CASES, ids=[f"{c[0]}-{c[1]}" for c in CASES])
def test_scheduled_depformer_matches_fp64_reference(member, name, mode, batches, sampled):
    cfg = MEMBERS[member]
    sd = synth_lm_state_dict(cfg, seed=41, device="cuda")
    lm = _model(cfg, sd, mode)
    try:
        failures = _check(lm, cfg, sd, f"{member} {name}", batches, sampled, {}, len(name) * 7 + len(member))
    finally:
        del lm
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("member,name,batches,sampled,opt", CASES_OPT, ids=[f"{c[0]}-{c[1]}" for c in CASES_OPT])
def test_scheduled_depformer_under_guidance_and_int8(member, name, batches, sampled, opt):
    cfg = MEMBERS[member]
    if opt.get("int8"):
        cfg = dataclasses.replace(cfg, quantize=True)
    sd = synth_lm_state_dict(cfg, seed=43, device="cuda")
    if opt.get("int8"):
        sd = dep_row_scaled(sd, seed=5)
    lm = _model(cfg, sd)
    try:
        failures = _check(lm, cfg, sd, f"{member} {name}", batches, sampled, opt, len(name) * 11)
    finally:
        del lm
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


def test_setters_refuse_once_tensors_are_loaded():
    from moshi_b200.models.lm import _config_struct
    import ctypes as C
    L, cfg = _lib.lib(), tiny_lm_config()
    h = C.c_void_p()
    _lib.check(L.b200_lm_create(C.byref(_config_struct(cfg)), C.byref(h)))
    try:
        t = torch.ones(1, 1, cfg.depformer_dim, device="cuda", dtype=torch.bfloat16)
        shape = (C.c_int64 * 3)(*t.shape)
        _lib.check(L.b200_lm_load_tensor(h, b"depformer.layers.0.norm1.alpha", _lib.ptr(t), _lib.B200_BF16, 3, shape))
        assert L.b200_lm_set_depformer_schedule(h, (C.c_int * 8)(*range(8)), 8) == _lib.B200_ERR_STATE
        assert L.b200_lm_set_depformer_low_rank(h, 8) == _lib.B200_ERR_STATE
    finally:
        L.b200_lm_destroy(h)


def _used_by_model(cfg, sd) -> int:
    from moshi_b200.models import LMModel
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    lm = LMModel(cfg, sd, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    used = free0 - torch.cuda.mem_get_info()[0]
    del lm
    torch.cuda.empty_cache()
    return used


def test_shared_weight_sets_are_resident_once():
    sched = MEMBERS["7b"]
    plain = dataclasses.replace(sched, depformer_weights_per_step_schedule=None)
    n_sets, dd, d, F = sched.depformer_n_sets, sched.depformer_dim, sched.dim, sched.depformer_ffn_hidden
    per_set = (dd * d + sched.depformer_num_layers * (4 * dd * dd + 3 * F * dd)) * 2
    want = (sched.dep_q - n_sets) * per_set
    used = {}
    for name, cfg in (("plain", plain), ("sched", sched)):
        sd = synth_lm_state_dict(cfg, seed=3, device="cuda")
        used[name] = _used_by_model(cfg, sd)
        del sd
    saved = used["plain"] - used["sched"]
    print(f"\ndevice memory after load: unscheduled {used['plain'] / 2**20:.1f} MiB, scheduled {used['sched'] / 2**20:.1f} MiB, "
          f"saved {saved / 2**20:.1f} MiB, {sched.dep_q - n_sets} weight sets = {want / 2**20:.1f} MiB")
    assert 0.95 * want <= saved <= 1.1 * want


@torch.no_grad()
def test_session_move_and_state_round_trip_continue_bit_for_bit():
    from moshi_b200.models import LMGen
    cfg = MEMBERS["7b"]
    sd = synth_lm_state_dict(cfg, seed=47, device="cuda")
    lm = _model(cfg, sd)
    B, warm, after = 3, 4, 3
    g = torch.Generator().manual_seed(5)
    codes = torch.randint(0, cfg.card, (warm + after, B, cfg.n_q - cfg.dep_q, 1), generator=g).cuda()
    kt, ka = SMP["top_k_text"], min(SMP["top_k"], cfg.card)
    noise = torch.empty(warm + after, B, kt + cfg.dep_q * ka).exponential_(1, generator=g).cuda()

    swap = [2, 1, 0]

    def run(move):
        gen = LMGen(lm, use_sampling=True, **SMP)
        outs = []
        perm = list(range(B))
        with gen.streaming(B):
            for i in range(warm):
                gen.step(codes[i], noise=noise[i])
            if move == "state":
                st = gen.get_streaming_state()
                gen.step(codes[0], noise=noise[0])            # a step the restored state forgets
                gen.set_streaming_state(st)
            elif move == "session":                           # sessions 0 and 2 trade rows
                r0, r2 = gen.export_session(0), gen.export_session(2)
                gen.import_session(0, r2)
                gen.import_session(2, r0)
                perm = swap
            for i in range(warm, warm + after):
                o = gen.step(codes[i][perm].contiguous(), noise=noise[i][perm].contiguous())
                outs.append(o[perm].cpu())
                outs.append(gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card))[:, perm].cpu())
        return outs
    try:
        base = run(None)
        for move in ("state", "session"):
            got = run(move)
            assert all(torch.equal(a, b) for a, b in zip(base, got)), move
    finally:
        del lm
        torch.cuda.empty_cache()


@torch.no_grad()
@pytest.mark.parametrize("run,sampling", [("greedy", False), ("sampled", True)])
def test_reference_fixture(golden_dir, run, sampling):
    from moshi_b200.models import LMGen
    from tests.test_gpu_lm import _reference_trajectory
    info = json.loads((golden_dir / "lm_tiny_sched.json").read_text())
    gold = load_file(golden_dir / "lm_tiny_sched.safetensors")
    cfg = tiny_lm_config(depformer_weights_per_step_schedule=info["schedule"], depformer_low_rank_embeddings=info["low_rank"])
    sd = synth_lm_state_dict(cfg, seed=info["seed"])
    B, steps, codes = info["B"], info["steps"], gold["codes"]
    lm = _model(cfg, sd)
    gen = LMGen(lm, use_sampling=sampling, temp=0.8, temp_text=0.7)
    orc = LMOracle(sd, sched_spec(cfg), use_sampling=sampling, tie_break="index")
    orc.streaming(B)
    torch.manual_seed(info["noise_seed"])
    rec, worst, match, total, samp_bad = [], 0.0, 0, 0, 0
    with gen.streaming(B):
        for i in range(steps):
            scenarios.lm_mask_events(gen, i, B)
            scenarios.lm_mask_events(orc, i, B)
            nt, na = scenarios.lm_noise(cfg, B) if sampling else (None, None)
            dbg: dict = {}
            want = orc.step(codes[i], nt, na, debug=dbg)
            got = gen.step(codes[i].cuda(), noise=gen.pack_noise(nt, na) if sampling else None)
            assert (want is None) == (got is None), i
            live = orc.exec_mask
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu()
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            worst = max(worst, float((tl - dbg["text_logits"].float()[:, 0, 0])[live].abs().max()))
            if sampling:
                samp_bad += int((sample_token(tl, True, 0.7, 25, nt, "index") != tt)[live].sum())
                for k in range(cfg.dep_q):
                    samp_bad += int((sample_token(dl[k], True, 0.8, 250, na[k], "index") != at[k])[live].sum())
            rec.append((live.clone(), torch.cat([tt[:, None], at.t()], 1), [tl] + [dl[k] for k in range(cfg.dep_q)],
                        torch.cat([dbg["text_token"][:, None], dbg["audio_tokens"]], 1)))
            if got is not None:
                ok = (got.cpu() == want)[live]
                match += int(ok.sum())
                total += ok.numel()
            pos = orc.offsets % orc.cache.shape[2]              # keep the oracle on the handle's trajectory
            for b in range(B):
                if live[b]:
                    orc.cache[b, 0, pos[b]] = tt[b]
                    orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print(f"\n{run}: worst text logit difference {worst:.3e}, tokens equal to the oracle {match}/{total}, "
          f"sampler mismatches {samp_bad}")
    assert worst < LOGIT_ATOL
    assert samp_bad == 0
    if not sampling:
        assert match / total > 0.97
        compared, unexcused = _reference_trajectory(cfg, rec, gold[f"{run}.tokens"], {20: (1,)})
        print(f"against the reference fixture: {compared} tokens compared on its trajectory, {unexcused} unexcused")
        assert compared > 0 and unexcused == 0
