"""GPU: the Exp(1) noise the LM step draws itself, from the Philox bits to the sampled tokens.

Every caller that serves traffic passes no noise (``LMGen.step(noise=None)``, the frame service, bench.py): the step then
draws it inside its own graph (``lm_noise_kernel``: Philox4x32-10 keyed by the session seed, counter (element / 4, step)),
and ``lm_finish_kernel`` advances the step counter.  This file holds that path to the host reference of tests/util.py
(``step_noise_ref``, checked against the published Philox known answers by tests/test_philox_cpu.py):

* the raw draws bit for bit, at every length, seed and counter edge, and nothing written past the end;
* the bits -> Exp(1) transform over all 2^24 patterns: finite, strictly positive, non-increasing, within 2 fp32 ulp of fp64;
* the LM step with ``noise=None``: at every step the noise it drew equals the reference for (seed, step), and every token is
  what the reference sampler draws from the device's own logits with that noise, on every depformer path, eager and graphed,
  at 1 to 129 sessions, under CFG (B rows of noise, not 2B), with a paused row and on the STT configuration;
* reproducibility: torch.manual_seed, a snapshot restored mid-run, and b200_lm_seed_noise restarting the counter;
* the distribution of sampled tokens (chi-square against fp64 top-k probabilities) and of the raw draws (KS against Exp(1)).
The seeds are fixed, so every verdict is deterministic.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import LMConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict
from oracle import scenarios
from tests.util import cptr, exp1_ref64, f32_ulp, sampler_mismatches, step_noise_ref, step_words

pytestmark = pytest.mark.gpu

AUTO, CHAIN, FUSED = _lib.B200_DEPFORMER_AUTO, _lib.B200_DEPFORMER_CHAIN, _lib.B200_DEPFORMER_FUSED

SMP = dict(temp=0.8, top_k=250, temp_text=0.7, top_k_text=25)     # LMGen's defaults: 25 + 8 x 250 = 2025 draws per row


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    return _lib.lib()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lm_noise(lib, n: int, seed: int, ctr: int, pad: int = 0) -> torch.Tensor:
    """b200_op_lm_noise into a NaN-poisoned buffer of n + pad floats (returned whole, on the host)."""
    from moshi_b200 import _lib
    out = torch.full((n + pad,), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_op_lm_noise(cptr(out), n, C.c_uint64(seed), C.c_uint64(ctr), _stream()))
    torch.cuda.synchronize()
    return out.cpu()


def _exp1(lib, words: np.ndarray) -> torch.Tensor:
    """b200_op_exp1 on host uint32 words -> fp32 on the host."""
    from moshi_b200 import _lib
    w = torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint32).view(np.int32)).cuda()
    out = torch.full((w.numel(),), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(lib.b200_op_exp1(cptr(w), cptr(out), w.numel(), _stream()))
    torch.cuda.synchronize()
    return out.cpu()


def _ulps(got: np.ndarray, want64: np.ndarray) -> np.ndarray:
    return np.abs(got.astype(np.float64) - want64) / f32_ulp(want64)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the raw draws
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 2 ** 62 - 1, 0xDEADBEEF_00000001], ids=["zero", "2^62-1", "high-word"])
def test_lm_noise_equals_host_reference(lib, seed):
    """Every element bit for bit the transform of the host reference's word, within 2 ulp of fp64, nothing past n."""
    worst = 0.0
    for ctr in (0, 1, 2 ** 32 + 5):
        for n in (1, 3, 5, 2025, 40 * 2025, 2 ** 22 + 3):
            got = _lm_noise(lib, n, seed, ctr, pad=9)
            assert torch.isnan(got[n:]).all(), f"seed {seed:#x} ctr {ctr} n {n}: elements past n were written"
            got = got[:n].numpy()
            words = step_words(seed, ctr, n)
            want = _exp1(lib, words).numpy()
            bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
            assert bad.size == 0, (f"seed {seed:#x} ctr {ctr} n {n}: {bad.size} elements differ from the transform of the "
                                   f"reference's words, first {bad[:8].tolist()}")
            m, ref = step_noise_ref(seed, ctr, n)
            top = m == (1 << 24) - 1                   # u = 1: fp64 gives 0, the transform 2^-24
            assert (got[top] == 2.0 ** -24).all(), f"seed {seed:#x} ctr {ctr} n {n}: the top pattern gave {got[top]}"
            if (~top).any():
                u = _ulps(got[~top], ref[~top])
                worst = max(worst, float(u.max()))
                assert u.max() <= 2, f"seed {seed:#x} ctr {ctr} n {n}: {int((u > 2).sum())} elements beyond 2 ulp of fp64"
    print(f"\nseed {seed:#x}: worst distance to fp64 {worst:.3f} ulp")


# ---------------------------------------------------------------------------------------------------------------------------
# 2. the transform, every input
# ---------------------------------------------------------------------------------------------------------------------------
def test_exp1_every_pattern(lib):
    """All 2^24 patterns m = r >> 8, with random low bits (which the transform must ignore): every output finite with its
    sign bit clear and above zero, non-increasing in m, within 2 fp32 ulp of fp64 -log((m + 1) / 2^24) below the top
    pattern, and the top pattern (u = 1) positive and no larger than the next one."""
    m = np.arange(1 << 24, dtype=np.uint32)
    low = np.random.default_rng(9).integers(0, 256, size=m.size, dtype=np.uint32)
    got = _exp1(lib, (m << np.uint32(8)) | low).numpy()
    bare = _exp1(lib, m << np.uint32(8)).numpy()
    assert np.array_equal(got.view(np.uint32), bare.view(np.uint32)), "the low 8 bits changed a draw"
    nonpos = np.flatnonzero(~(got > 0) | np.signbit(got) | ~np.isfinite(got))
    worst = _ulps(got[:-1], exp1_ref64(m[:-1]))
    rises = np.flatnonzero(np.diff(got.astype(np.float64)) > 0)
    print(f"\nexp1: {nonpos.size} patterns not finite and positive {[(int(i), float(got[i])) for i in nonpos[:8]]}; "
          f"{rises.size} rises; worst {worst.max():.3f} ulp at m = {int(worst.argmax())}; top two {got[-1]!r}, {got[-2]!r}")
    assert nonpos.size == 0, f"patterns giving 0, a negative or a non-finite draw: {[(int(i), float(got[i])) for i in nonpos[:16]]}"
    assert rises.size == 0, f"the draw rises with m at {rises[:16].tolist()}"
    assert worst.max() <= 2, f"{int((worst > 2).sum())} patterns beyond 2 ulp of fp64, first {np.flatnonzero(worst > 2)[:8].tolist()}"
    assert 0 < got[-1] <= got[-2]


# ---------------------------------------------------------------------------------------------------------------------------
# 3. the LM step with noise=None
# ---------------------------------------------------------------------------------------------------------------------------
_sd_cache: dict = {}


def _member(name: str):
    if name not in _sd_cache:
        if name == "stt":
            cfg = LMConfig.from_dict(scenarios.stt_reference_kwargs())
            sd = scenarios.stt_state_dict()
        else:
            cfg = tiny_lm_config(card=2048)            # 2048-entry audio vocabulary: top-250 of the 7B, 2025 draws per row
            sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
        _sd_cache[name] = (cfg, sd)
    return _sd_cache[name]


def _model(cfg: LMConfig, sd: dict, mode: int):
    """LMModel whose depformer runs in ``mode`` (b200_lm_set_depformer)."""
    from moshi_b200.models import LMModel
    lm = LMModel(cfg, sd, device="cuda")
    _lib.check(_lib.lib().b200_lm_set_depformer(lm._h, mode))
    return lm


# (member, depformer path, depformer mode, batch sizes, CFG coefficient).  At 1 and 2 sessions the default depformer is the
# GEMV chain; "fused-forced" runs the persistent kernel there.  CFG doubles the model rows, so its batches stay at <= 128.
STEP_CASES = [
    ("tiny", "fused", AUTO, (3, 40, 129), 1.0),
    ("tiny", "chain", CHAIN, (3, 40, 129), 1.0),
    ("tiny", "gemv", AUTO, (1,), 1.0),
    ("tiny", "fused-forced", FUSED, (1,), 1.0),
    ("tiny", "fused-cfg", AUTO, (3, 40), 3.0),
    ("tiny", "chain-cfg", CHAIN, (3,), 3.0),
    ("stt", "none", AUTO, (1, 3, 40), 1.0),
]
STEPS = 5
SEED = 0x5EED_0000_0000_0001 + 2 ** 40


def _check_steps(lib, lm, cfg, B: int, graph: bool, cfg_coef: float, g: torch.Generator) -> dict:
    """Steps with noise=None from a known seed; per step: the step's noise against the reference, every executing row's
    tokens against the reference sampler on the device's own logits with that noise."""
    from moshi_b200 import _lib
    from moshi_b200.models import LMGen
    gen = LMGen(lm, use_sampling=True, cfg_coef=cfg_coef, cfg_is_no_text=cfg_coef != 1.0, **SMP)
    gen.use_graph = graph
    Q = cfg.dep_q
    kt, ka = min(SMP["top_k_text"], cfg.text_card), min(SMP["top_k"], cfg.card)
    npr = kt + Q * ka
    res = dict(noise_bad=0, sampler=0, decisions=0, not_argmax=0)
    paused = B // 2 if B > 1 else None
    with gen.streaming(B):
        assert gen._noise_per_row == npr
        _lib.check(lib.b200_lm_seed_noise(gen._h, C.c_uint64(SEED)))
        for step in range(STEPS):
            ex = torch.ones(B, dtype=torch.bool)
            if paused is not None and step in (2, 3):
                ex[paused] = False
            gen.set_exec_mask(ex.cuda())
            codes = torch.randint(0, cfg.card, (B, cfg.n_q - Q, 1), generator=g).cuda()
            gen.step(codes)
            noise = gen.read_buffer("noise", torch.float32, (B, npr))
            want = _exp1(lib, step_words(SEED, step, B * npr)).reshape(B, npr)
            res["noise_bad"] += int((noise.cpu().view(torch.int32) != want.view(torch.int32)).sum())
            rows = ex.nonzero().flatten().cuda()
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card))
            text = gen.read_buffer("text_token", torch.int64, (B,))
            pairs = [(tl, text, SMP["temp_text"], SMP["top_k_text"], noise[:, :kt])]
            if Q:
                dl = gen.read_buffer("dep_logits", torch.bfloat16, (Q, B, cfg.card))
                toks = gen.read_buffer("audio_tokens", torch.int64, (Q, B))
                pairs += [(dl[k], toks[k], SMP["temp"], SMP["top_k"], noise[:, kt + k * ka:kt + (k + 1) * ka]) for k in range(Q)]
            for lg, tk, temp, top_k, nz in pairs:
                lg, tk, nz = lg[rows], tk[rows], nz[rows]
                res["sampler"] += sampler_mismatches(lg, tk, True, temp, top_k, nz)
                res["decisions"] += rows.numel()
                res["not_argmax"] += int((tk != lg.float().argmax(-1)).sum())
    return res


@pytest.mark.parametrize("member,path,mode,batches,cfg_coef", STEP_CASES, ids=[f"{c[0]}-{c[1]}" for c in STEP_CASES])
def test_step_draws_its_noise_and_samples_with_it(lib, member, path, mode, batches, cfg_coef):
    cfg, sd = _member(member)
    lm = _model(cfg, sd, mode)
    g = torch.Generator().manual_seed(17)
    failures = []
    try:
        for B in batches:
            for graph in (False, True):
                r = _check_steps(lib, lm, cfg, B, graph, cfg_coef, g)
                tag = f"{member} {path} B={B} graph={graph} cfg={cfg_coef}"
                print(f"\n{tag}: noise elements off {r['noise_bad']}, sampler mismatches {r['sampler']}/{r['decisions']}, "
                      f"tokens other than the argmax {r['not_argmax']}")
                if r["noise_bad"] or r["sampler"]:
                    failures.append(f"{tag}: {r['noise_bad']} noise elements differ from the reference, "
                                    f"{r['sampler']} tokens differ from the reference sampler")
                if r["not_argmax"] == 0:
                    failures.append(f"{tag}: every token was the argmax: nothing was sampled")
    finally:
        del lm
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------------------------------
# 4. reproducibility and state
# ---------------------------------------------------------------------------------------------------------------------------
def _tokens(gen, cfg, B) -> torch.Tensor:
    text = gen.read_buffer("text_token", torch.int64, (B,))
    audio = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B))
    return torch.cat([text[None], audio]).cpu()


def _stream_tokens(gen, cfg, B, codes) -> list:
    out = []
    for c in codes:
        gen.step(c.cuda())
        out.append(_tokens(gen, cfg, B))
    return out


@pytest.mark.parametrize("graph", [False, True])
def test_step_noise_is_reproducible_and_restorable(lib, graph):
    from moshi_b200 import _lib
    from moshi_b200.models import LMGen
    cfg, sd = _member("tiny")
    lm = _model(cfg, sd, AUTO)
    B, n = 5, 8
    g = torch.Generator().manual_seed(23)
    codes = [torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g) for _ in range(n)]

    def run(seed):
        gen = LMGen(lm, use_sampling=True, **SMP)
        gen.use_graph = graph
        torch.manual_seed(seed)
        with gen.streaming(B):
            return _stream_tokens(gen, cfg, B, codes)

    a, b, c = run(1), run(1), run(2)
    assert all(torch.equal(x, y) for x, y in zip(a, b)), "the same torch.manual_seed gave another token stream"
    assert any(not torch.equal(x, y) for x, y in zip(a, c)), "another torch.manual_seed gave the same token stream"

    # a snapshot taken mid-run and restored continues exactly like the uninterrupted run
    gen = LMGen(lm, use_sampling=True, **SMP)
    gen.use_graph = graph
    torch.manual_seed(1)
    with gen.streaming(B):
        first = _stream_tokens(gen, cfg, B, codes[:4])
        snap = gen.get_streaming_state()
        assert int(snap[""].noise_counter.reshape(-1)[0]) == 4
        rest = _stream_tokens(gen, cfg, B, codes[4:])
        assert all(torch.equal(x, y) for x, y in zip(first + rest, a))
        gen.set_streaming_state(snap)
        again = _stream_tokens(gen, cfg, B, codes[4:])
        assert all(torch.equal(x, y) for x, y in zip(again, rest)), "the continuation from the snapshot differs"

        # b200_lm_seed_noise restarts the counter: the next step draws step 0 of the new seed
        npr = gen._noise_per_row
        _lib.check(lib.b200_lm_seed_noise(gen._h, C.c_uint64(SEED)))
        assert int(gen.get_streaming_state()[""].noise_counter.reshape(-1)[0]) == 0
        for step in range(2):
            gen.step(codes[step].cuda())
            noise = gen.read_buffer("noise", torch.float32, (B, npr)).cpu()
            want = _exp1(lib, step_words(SEED, step, B * npr)).reshape(B, npr)
            assert torch.equal(noise.view(torch.int32), want.view(torch.int32)), f"step {step} after seeding"
    del gen, lm
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------
# 6. distributions
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("card,k,temp", [(2048, 250, 0.8), (32000, 25, 0.7)])
def test_sampled_tokens_follow_the_top_k_distribution(lib, card, k, temp):
    """2^20 samples of one logit row, each with its own draws from b200_op_lm_noise, against fp64 p_j / sum_top-k p by
    chi-square, bins pooled so that each expects at least 5."""
    from scipy import stats as sps
    from moshi_b200 import _lib
    g = torch.Generator().manual_seed(card + k)
    logits = (torch.randn(card, generator=g) * 2.0).bfloat16()
    lg = logits.double()
    order = torch.sort(lg, descending=True, stable=True).indices[:k]
    p = torch.softmax(lg / temp, -1)[order]
    expect_p = (p / p.sum()).numpy()
    rows, total = 4096, 1 << 20
    dev_logits = logits.cuda()[None].expand(rows, card).contiguous()
    out = torch.empty(rows, dtype=torch.int64, device="cuda")
    counts = torch.zeros(card, dtype=torch.int64, device="cuda")
    for chunk in range(total // rows):
        noise = torch.empty(rows * k, dtype=torch.float32, device="cuda")
        _lib.check(lib.b200_op_lm_noise(cptr(noise), rows * k, C.c_uint64(0xC0FFEE + card), C.c_uint64(chunk), _stream()))
        _lib.check(lib.b200_op_sample(cptr(dev_logits), cptr(noise), cptr(out), rows, card, 1, temp, k, _stream()))
        counts += torch.bincount(out, minlength=card)
    counts = counts.cpu()
    assert int(counts.sum()) == total
    outside = int(counts.sum() - counts[order].sum())
    assert outside == 0, f"{outside} samples outside the top {k}"
    obs = counts[order].numpy().astype(np.float64)
    exp = expect_p * total
    keep = exp >= 5
    o, e = list(obs[keep]), list(exp[keep])
    if (~keep).any():
        po, pe = obs[~keep].sum(), exp[~keep].sum()
        if pe >= 5:
            o.append(po); e.append(pe)
        else:
            i = int(np.argmin(e)); o[i] += po; e[i] += pe
    chi = sps.chisquare(np.array(o), np.array(e) * (sum(o) / sum(e)))
    print(f"\ncard {card} k {k} temp {temp}: {len(o)} bins, chi2 {chi.statistic:.1f}, p = {chi.pvalue:.3g}")
    assert chi.pvalue > 1e-6


def test_raw_draws_are_exp1(lib):
    """2^24 draws of one step against Exp(1) by a Kolmogorov-Smirnov test."""
    from scipy import stats as sps
    x = _lm_noise(lib, 1 << 24, 0x0BADC0DE_12345678, 7).double().numpy()
    ks = sps.kstest(x, "expon")
    print(f"\nKS of 2^24 draws against Exp(1): D = {ks.statistic:.3g}, p = {ks.pvalue:.3g}; mean {x.mean():.6f}, min {x.min():.3g}")
    assert x.min() > 0
    assert ks.pvalue > 1e-6
