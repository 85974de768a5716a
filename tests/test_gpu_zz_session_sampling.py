"""GPU: per-session sampling settings (b200_lm_set_session_sampling / b200_lm_set_row_sampling).

1. the text sampler at op level against the numpy restatement of tests/test_session_sampling_cpu.py, and its fp32-score
   instantiation against the bf16 sampler on rows with default settings, bit for bit;
2. a session-sampling handle whose rows follow the handle-wide values steps the same tokens as a plain handle;
3. rows are independent: row j of a mixed batch equals row j of a batch where every row has row j's settings;
4. the whole step against the restatement on the device's own guided text logits, history and noise, with wrap, pauses, reset;
5. state entries and session records: round trips, moves, refusals;
6. the dialogue service: slots at different settings equal uniform services slot by slot.
The restatement's softmax sum is not the device's, so a sampled row whose two best ranks lie within 1e-5 of each other is
excused (and counted); everything else is compared token for token.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict
from oracle import scenarios
from tests.test_session_sampling_cpu import settings, text_sample_ref
from tests.util import cptr

pytestmark = pytest.mark.gpu

AUTO, CHAIN, FUSED = _lib.B200_DEPFORMER_AUTO, _lib.B200_DEPFORMER_CHAIN, _lib.B200_DEPFORMER_FUSED


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _row_struct(st: dict) -> _lib.RowSamplingC:
    return _lib.RowSamplingC(**st)


def _random_settings(rng, n: int, top_k: int, greedy_share: float = 0.2) -> list:
    out = []
    for _ in range(n):
        out.append(settings(temp_text=0.0 if rng.random() < greedy_share else float(rng.uniform(0.3, 1.5)), temp=float(rng.uniform(0.3, 1.2)),
                            top_k_text=int(rng.integers(1, top_k + 1)), top_k=int(rng.integers(1, top_k + 1)),
                            pad_mult=float(rng.choice([0.0, rng.uniform(-3, 3)])), repetition_context=int(rng.choice([0, 1, 7, 64, 200])),
                            repetition_penalty=float(rng.choice([1.0, rng.uniform(1.05, 2.0), rng.uniform(0.5, 0.95)]))))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# 1. op level
# ---------------------------------------------------------------------------------------------------------------------------
def _op_text(lib, logits_bf16, noise, ring, count, use_sampling, temp, top_k, sts):
    B, card = logits_bf16.shape
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    ring_d, count_d = torch.from_numpy(ring).cuda(), torch.from_numpy(count.astype(np.int32)).cuda()
    p = None if sts is None else (_lib.RowSamplingC * B)(*[_row_struct(s) for s in sts])
    _lib.check(lib.b200_op_sample_text_rows(cptr(logits_bf16), cptr(noise), noise.shape[1], cptr(out), B, card, int(use_sampling),
                                            C.c_float(temp), top_k, p, cptr(ring_d), cptr(count_d), ring.shape[1], _stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), ring_d.cpu().numpy(), count_d.cpu().numpy()


@pytest.mark.parametrize("card", [500, 32000, 48000])
@pytest.mark.parametrize("top_k", [1, 25, 250, 1024])
def test_op_text_sampler_equals_restatement(lib, card, top_k):
    rng = np.random.default_rng(card * 7 + top_k)
    B, N = 48, 64
    logits = (torch.from_numpy(rng.standard_normal((B, card)).astype(np.float32)) * 3).to(torch.bfloat16).cuda()
    noise = torch.from_numpy(rng.exponential(size=(B, top_k)).astype(np.float32)).cuda()
    ring = rng.integers(0, min(card + 1, 600), size=(B, N)).astype(np.int32)          # small ids: repeats, and some special ids
    count = rng.integers(0, 3 * N, size=B).astype(np.int64)
    sts = _random_settings(rng, B, top_k)
    got, ring_g, count_g = _op_text(lib, logits, noise, ring, count, True, 0.7, top_k, sts)
    want, stable, ring_w, count_w = text_sample_ref(logits.float().cpu().numpy(), noise.cpu().numpy(), ring, count, True, 0.7, top_k, sts)
    bad = np.flatnonzero((got != want) & stable)
    assert bad.size == 0, f"rows {bad.tolist()}: device {got[bad].tolist()} restatement {want[bad].tolist()}"
    same = got == want
    assert np.array_equal(count_g[same], count_w[same]) and np.array_equal(ring_g[same], ring_w[same])
    print(f"\ncard {card} top_k {top_k}: {int((~stable).sum())} near-tie rows excused, {int((got != want).sum())} differ")

    # default settings: the fp32-score instantiation picks what the bf16 sampler picks, for sampled and greedy handles
    # (b200_op_sample's noise rows are min(top_k, card) floats long)
    nz = noise[:, :min(top_k, card)].contiguous()
    for use_sampling in (True, False):
        plain = torch.empty(B, dtype=torch.int64, device="cuda")
        _lib.check(lib.b200_op_sample(cptr(logits), cptr(nz), cptr(plain), B, card, int(use_sampling), C.c_float(0.7), top_k, _stream()))
        rows, _, _ = _op_text(lib, logits, nz, ring, count, use_sampling, 0.7, top_k, None)
        assert np.array_equal(rows, plain.cpu().numpy()), f"use_sampling={use_sampling}: the two instantiations differ"


def test_op_text_sampler_refuses_out_of_range(lib):
    B, card = 2, 500
    logits = torch.zeros(B, card, dtype=torch.bfloat16, device="cuda")
    noise = torch.ones(B, 25, device="cuda")
    ring, count = np.zeros((B, 4), np.int32), np.zeros(B, np.int64)
    for bad in (dict(top_k_text=26), dict(temp_text=-1.0), dict(repetition_penalty=0.0), dict(repetition_context=2000)):
        st = settings(top_k=25)
        st.update(bad)
        with pytest.raises(ValueError):
            _op_text(lib, logits, noise, ring, count, True, 0.7, 25, [st, st])


# ---------------------------------------------------------------------------------------------------------------------------
# helpers for the step tests
# ---------------------------------------------------------------------------------------------------------------------------
_sd: dict = {}


def _cfg_sd(text_card: int = 500):
    if text_card not in _sd:
        cfg = tiny_lm_config(text_card=text_card)
        _sd[text_card] = (cfg, synth_lm_state_dict(cfg, seed=scenarios.LM_SEED))
    return _sd[text_card]


def _model(text_card: int, mode: int):
    from moshi_b200.models import LMModel
    cfg, sd = _cfg_sd(text_card)
    lm = LMModel(cfg, sd, device="cuda")
    _lib.check(_lib.lib().b200_lm_set_depformer(lm._h, mode))
    return lm


def _gen(lm, B, history, use_sampling=True, cfg_coef=1.0, **kw):
    from moshi_b200.models import LMGen
    g = LMGen(lm, use_sampling=use_sampling, cfg_coef=cfg_coef, cfg_is_no_text=cfg_coef != 1.0, **kw)
    g.session_sampling = history
    g.streaming_forever(B)
    return g


def _run(gen, codes, noises, events=None):
    """Steps gen through codes [T, B, K, 1] with noise [T, B, n]; events: {step: ("exec", mask) | ("reset", mask)}."""
    outs = []
    for i in range(codes.shape[0]):
        ev = (events or {}).get(i)
        if ev is not None:
            kind, m = ev
            if kind == "exec":
                gen.set_exec_mask(m.cuda())
            else:
                gen.reset_streaming(m.cuda())
        gen.step(codes[i].cuda(), noise=None if noises is None else noises[i])
        outs.append(torch.cat([gen.read_buffer("text_token", torch.int64, (gen._batch,))[:, None],
                               gen.read_buffer("audio_tokens", torch.int64, (gen.lm_model.dep_q, gen._batch)).t()], 1).cpu())
    return torch.stack(outs)


def _inputs(cfg, B, T, npr, seed):
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, cfg.card, (T, B, cfg.n_q, 1), generator=g)
    noises = torch.empty(T, B, npr).exponential_(1, generator=g).cuda()
    return codes, noises


def _events(B, T):
    ex = torch.ones(B, dtype=torch.bool)
    ex[B // 2] = False
    rs = torch.zeros(B, dtype=torch.bool)
    rs[0] = True
    return {T // 4: ("exec", ex), T // 2: ("exec", torch.ones(B, dtype=torch.bool)), 3 * T // 4: ("reset", rs)}


# ---------------------------------------------------------------------------------------------------------------------------
# 2. on with defaults equals off
# ---------------------------------------------------------------------------------------------------------------------------
DEFAULT_CASES = [(500, B, mode, 1.0) for B in (1, 2, 3, 40, 130) for mode in (CHAIN, FUSED) if not (mode == FUSED and B == 130)]
DEFAULT_CASES += [(500, 3, AUTO, 3.0), (48000, 3, AUTO, 1.0), (48000, 40, AUTO, 1.0)]


@pytest.mark.parametrize("text_card,B,mode,cfg_coef", DEFAULT_CASES)
@pytest.mark.parametrize("use_sampling", [False, True])
def test_defaults_equal_plain_handle(text_card, B, mode, cfg_coef, use_sampling):
    T = 40
    lm_a, lm_b = _model(text_card, mode), _model(text_card, mode)
    cfg = lm_a.cfg
    plain, ss = _gen(lm_a, B, None, use_sampling, cfg_coef), _gen(lm_b, B, 16, use_sampling, cfg_coef)
    ss.set_session_sampling([0])                               # explicitly returned to the handle-wide values
    codes, noises = _inputs(cfg, B, T, plain._noise_per_row, seed=B + text_card)
    a = _run(plain, codes, noises if use_sampling else None, _events(B, T))
    b = _run(ss, codes, noises if use_sampling else None, _events(B, T))
    assert torch.equal(a, b), f"first difference at step {int((a != b).any(-1).any(-1).nonzero()[0])}"


# ---------------------------------------------------------------------------------------------------------------------------
# 3. rows are independent
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [CHAIN, FUSED])
def test_rows_are_independent(mode):
    B, T = 4, 30
    rng = np.random.default_rng(5)
    sts = _random_settings(rng, B, 25, greedy_share=0.25)
    for st in sts:
        st["top_k"] = int(rng.integers(1, 251))
        st["repetition_context"] = max(st["repetition_context"], 7)
        st["repetition_penalty"] = 1.6
    lm = _model(500, mode)
    cfg = lm.cfg
    mixed = _gen(lm, B, 32)
    for b, st in enumerate(sts):
        mixed.set_session_sampling([b], **st)
    codes, noises = _inputs(cfg, B, T, mixed._noise_per_row, seed=11)
    got = _run(mixed, codes, noises)
    mixed._stop()
    for j, st in enumerate(sts):
        uni = _gen(lm, B, 32)
        uni.set_session_sampling(list(range(B)), **st)
        want = _run(uni, codes, noises)
        uni._stop()
        assert torch.equal(got[:, j], want[:, j]), f"row {j}: differs from a batch at its settings"


# ---------------------------------------------------------------------------------------------------------------------------
# 4. the whole step against the restatement
# ---------------------------------------------------------------------------------------------------------------------------
def _read_hist(gen):
    st = gen.get_streaming_state()[""].session_sampling
    return st.history.cpu().numpy(), st.count.cpu().numpy().astype(np.int64), st.params.cpu().numpy()


@pytest.mark.parametrize("mode", [CHAIN, FUSED])
def test_step_text_tokens_equal_restatement(mode):
    B, T, N = 6, 60, 8
    lm = _model(500, mode)
    cfg = lm.cfg
    gen = _gen(lm, B, N)
    sts = [settings(temp_text=0.8, repetition_context=1, repetition_penalty=1.3),
           settings(temp_text=0.6, repetition_context=7, repetition_penalty=2.0, pad_mult=-1.0, top_k_text=10),
           settings(temp_text=0.0, repetition_context=200, repetition_penalty=1.7),
           settings(temp_text=1.0, repetition_context=200, repetition_penalty=1.5, pad_mult=2.0, top_k_text=1),
           None, settings(temp_text=0.9, repetition_context=7, repetition_penalty=1.9, top_k_text=25)]
    for b, st in enumerate(sts):
        if st is not None:
            gen.set_session_sampling([b], **st)
    codes, noises = _inputs(cfg, B, T, gen._noise_per_row, seed=3)
    events = _events(B, T)
    executed = np.ones(B, bool)
    excused = 0
    for i in range(T):
        ev = events.get(i)
        if ev is not None:
            kind, m = ev
            if kind == "exec":
                gen.set_exec_mask(m.cuda())
                executed = m.numpy().copy()
            else:
                gen.reset_streaming(m.cuda())
                executed[:] = True
                ring, count, params = _read_hist(gen)
                assert (count[m.numpy()] == 0).all(), "reset did not clear the history"
                assert (params[m.numpy(), 7] == (0 if sts[0] is None else 1)).all(), "reset changed the settings"
        ring, count, _ = _read_hist(gen)
        gen.step(codes[i].cuda(), noise=noises[i])
        tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu().numpy()
        tok = gen.read_buffer("text_token", torch.int64, (B,)).cpu().numpy()
        want, stable, ring_w, count_w = text_sample_ref(tl, noises[i].cpu().numpy(), ring, count, True, 0.7, 25, sts, executed)
        bad = np.flatnonzero((tok != want) & stable)
        assert bad.size == 0, f"step {i} rows {bad.tolist()}: device {tok[bad].tolist()} restatement {want[bad].tolist()}"
        excused += int((tok != want).sum())
        ring_g, count_g, _ = _read_hist(gen)
        ok = tok == want
        assert np.array_equal(count_g[ok], count_w[ok]) and np.array_equal(ring_g[ok], ring_w[ok]), f"step {i}: history"
    assert excused <= 2, f"{excused} near-tie tokens"
    assert (count > N).any(), "no history wrapped"


# ---------------------------------------------------------------------------------------------------------------------------
# 5. state and records
# ---------------------------------------------------------------------------------------------------------------------------
def test_state_round_trip_and_session_records():
    B, T = 3, 12
    lm = _model(500, AUTO)
    cfg = lm.cfg
    gen = _gen(lm, B, 16)
    gen.set_session_sampling([1], **settings(temp_text=0.9, repetition_context=7, repetition_penalty=1.8, pad_mult=1.0, top_k_text=20))
    codes, noises = _inputs(cfg, B, 2 * T, gen._noise_per_row, seed=21)
    _run(gen, codes[:T], noises[:T])
    snap = gen.get_streaming_state()
    assert snap[""].session_sampling.history.shape == (B, 16) and snap[""].session_sampling.params.shape == (B, 8)
    a = _run(gen, codes[T:], noises[T:])
    gen.set_session_sampling([0, 1, 2], temp_text=0.2)
    gen.set_streaming_state(snap)
    b = _run(gen, codes[T:], noises[T:])
    assert torch.equal(a, b), "the snapshot did not restore the settings and histories"

    # a session moved to another row of the same handle and to another handle of the same batch continues bit for bit
    gen.set_streaming_state(snap)
    rec = gen.export_session(1)
    other = _gen(_model(500, AUTO), B, 16)
    other.import_session(2, rec)
    gen.import_session(0, rec)
    c = _run(gen, codes[T:][:, [1, 1, 2]], noises[T:][:, [1, 1, 2]])
    d = _run(other, codes[T:][:, [0, 1, 1]], noises[T:][:, [0, 1, 1]])
    assert torch.equal(c[:, 0], a[:, 1]) and torch.equal(d[:, 2], a[:, 1]), "the moved session diverged"

    # refusals: feature on one side only, or another history length, with nothing written
    plain, n8 = _gen(_model(500, AUTO), B, None), _gen(_model(500, AUTO), B, 8)
    for g in (plain, n8):
        before = g.get_streaming_state()[""].cache.clone()
        with pytest.raises(ValueError):
            g.import_session(0, rec)
        assert torch.equal(g.get_streaming_state()[""].cache, before)
    with pytest.raises(ValueError):
        gen.import_session(0, plain.export_session(0))
    with pytest.raises(ValueError):
        gen.set_session_sampling([0], top_k_text=26)
    with pytest.raises(RuntimeError):
        plain.set_session_sampling([0], temp=0.5)


@pytest.mark.parametrize("mode", [CHAIN, FUSED])
def test_record_into_a_handle_with_smaller_top_k(mode):
    """A session whose settings were given on a handle with larger top-k values keeps sampling inside its noise block on a
    handle with smaller ones: its top-k values act as the handle's, exactly as if it had been given them there."""
    B, T = 3, 16
    st = settings(temp_text=0.9, temp=0.8, top_k_text=25, top_k=250, pad_mult=1.0, repetition_context=7, repetition_penalty=1.8)
    src = _gen(_model(500, mode), B, 16)
    src.set_session_sampling([1], **st)
    codes, noises = _inputs(src.lm_model.cfg, B, T, src._noise_per_row, seed=31)
    _run(src, codes[:T // 2], noises[:T // 2])
    rec = src.export_session(1)
    dst = _gen(_model(500, mode), B, 16, top_k=100, top_k_text=10)
    dst.import_session(0, rec)
    dst.import_session(1, rec)
    dst.set_session_sampling([1], **dict(st, top_k_text=10, top_k=100))
    assert dst._noise_per_row < src._noise_per_row
    _, nz = _inputs(dst.lm_model.cfg, B, T, dst._noise_per_row, seed=32)
    out = _run(dst, codes[T // 2:][:, [1, 1, 2]], nz[T // 2:][:, [0, 0, 2]])
    assert torch.equal(out[:, 0], out[:, 1]), "the imported row did not sample as one at the handle's top-k"
    assert dst.error_flags() == 0


# ---------------------------------------------------------------------------------------------------------------------------
# 6. the dialogue service
# ---------------------------------------------------------------------------------------------------------------------------
def test_dialogue_service_slots_equal_uniform_services():
    from moshi_b200.config import MimiConfig
    from moshi_b200.models import LMModel, MimiModel
    from moshi_b200.serving import ACTIVE, DialogueService
    from moshi_b200.synth import synth_mimi_state_dict
    B, T = 3, 10
    cfg = tiny_lm_config(card=2048)
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    msd = synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED)
    sts = [settings(temp_text=0.9, repetition_context=7, repetition_penalty=1.8),
           settings(temp_text=0.5, pad_mult=2.0, top_k_text=5, top_k=50, temp=1.1),
           settings(temp_text=0.0, repetition_context=200, repetition_penalty=1.4)]
    g = torch.Generator().manual_seed(4)
    pcm = (0.1 * torch.randn(T, B * 1920, generator=g)).numpy()
    npr = None

    def run(svc, change):
        nonlocal npr
        npr = npr or svc._lib.b200_lm_noise_per_row(svc.lm._h)
        gn = torch.Generator().manual_seed(8)
        outs = []
        for i in range(T):
            if i == T // 2:
                change(svc)
            noise = torch.empty(B, npr).exponential_(1, generator=gn).numpy()
            po, to, fl = np.zeros((B, 1920), np.float32), np.zeros((B, cfg.dep_q + 1), np.int64), np.zeros(B, np.uint8)
            svc.step(np.ascontiguousarray(pcm[i]), po, to, updates=[ACTIVE] * B, flags_out=fl, noise=noise)
            outs.append((po.copy(), to.copy()))
        svc.close()
        return outs

    def mk():
        return DialogueService(B, LMModel(cfg, sd, device="cuda"), MimiModel(MimiConfig(), msd, device="cuda"), session_sampling=32)

    mixed = mk()
    for b, st in enumerate(sts):
        mixed.set_session_sampling(b, **st)
    got = run(mixed, lambda s: s.set_session_sampling(0, **sts[1]))           # takes effect on the next frame
    for j in range(B):
        uni = mk()
        for b in range(B):
            uni.set_session_sampling(b, **sts[j])
        later = sts[1] if j == 0 else sts[j]
        want = run(uni, lambda s, later=later: [s.set_session_sampling(b, **later) for b in range(B)])
        for i in range(T):
            assert np.array_equal(got[i][1][j], want[i][1][j]) and np.array_equal(got[i][0][j], want[i][0][j]), f"slot {j} frame {i}"
