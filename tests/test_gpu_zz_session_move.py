"""GPU: moving one live session between rows, handles and GPUs (``LMGen.export_session`` / ``import_session``, the Mimi and
``DialogueService`` equivalents).  A moved session must continue bit for bit as it would have on its source: with the same
batch size the per-row results of the step do not depend on the row index, and the record carries the session's whole
per-row state."""
import numpy as np
import pytest
import torch

from moshi_b200.config import MimiConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict, synth_mimi_state_dict
from oracle import scenarios
from tests.util import greedy_unexcused

pytestmark = pytest.mark.gpu

STEPS_AFTER = 15
LAYOUTS = {
    "contig": {},
    "paged": {"kv_pool_frames": True},
    "int8": {"kv_dtype": "int8"},
    "e4m3": {"kv_dtype": "fp8_e4m3"},
}


@pytest.fixture(scope="module")
def tiny():
    cfg = tiny_lm_config()
    return cfg, synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)


@pytest.fixture(scope="module")
def lms(tiny):
    """Three handles of the tiny model: an LMGen streams on its model's handle, so concurrent sessions need one each."""
    from moshi_b200.models import LMModel
    cfg, sd = tiny
    return [LMModel(cfg, sd, device="cuda") for _ in range(3)]


_LIVE = []


@pytest.fixture(autouse=True)
def _stop_streaming():
    yield
    while _LIVE:
        _LIVE.pop()._stop()


def _lib():
    from moshi_b200 import _lib
    return _lib


def _gen(lm, B, sampling, layout="contig", cfg_coef=1.0, until=None, pool=None, capacity=None, page=4):
    from moshi_b200.models import LMGen
    gen = LMGen(lm, use_sampling=sampling, cfg_coef=cfg_coef, cfg_is_masked_until=until,
                cfg_is_no_text=cfg_coef != 1.0 and until is None)
    opts = LAYOUTS[layout]
    gen.kv_dtype = opts.get("kv_dtype", "bf16")
    if opts.get("kv_pool_frames"):
        gen.kv_pool_frames, gen.kv_page_slots = pool or (2 * B if cfg_coef != 1.0 else B) * lm.cfg.context, page
    elif pool is not None:
        gen.kv_pool_frames, gen.kv_page_slots = pool, page
    gen.kv_capacity = capacity
    gen.streaming_forever(B)
    _LIVE.append(gen)
    return gen


class Feed:
    """Codes and (sampled) noise of every step and row of one handle."""

    def __init__(self, cfg, gen, B, steps, sampling, seed):
        g = torch.Generator().manual_seed(seed)
        self.codes = torch.randint(0, cfg.card, (steps, B, cfg.n_q - cfg.dep_q, 1), generator=g)
        self.noise = torch.empty(steps, B, gen._noise_per_row).exponential_(1, generator=g) if sampling else None


def _step(gen, cfg, B, codes, noise):
    out = gen.step(codes.cuda(), noise=None if noise is None else noise.cuda())
    return (gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).cpu(),
            gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu(),
            None if out is None else out[:, :, 0].cpu())


def _same_row(x, i, y, j):
    assert torch.equal(x[0][i].view(torch.int16), y[0][j].view(torch.int16))
    assert torch.equal(x[1][:, i], y[1][:, j])
    assert (x[2] is None) == (y[2] is None)
    if x[2] is not None:
        assert torch.equal(x[2][i], y[2][j])


def _move_and_compare(lm_a, lm_b, lm_b0, cfg, B, src, dst, fill, sampling, i, j, extra=None, to=None):
    """A steps sessions for `fill` steps, B (and its twin B0) other sessions; A's row i moves into B's row j, whose session was
    live.  Then B's row j follows A's row i for STEPS_AFTER steps, and B's other rows follow B0."""
    steps = fill + STEPS_AFTER
    a = _gen(lm_a, B, sampling, src, **(extra or {}))
    b = _gen(lm_b, B, sampling, dst, **(extra or {}))
    b0 = _gen(lm_b0, B, sampling, dst, **(extra or {}))
    fa, fb = Feed(cfg, a, B, steps, sampling, 1), Feed(cfg, b, B, steps, sampling, 2)
    for t in range(fill):
        for gen, f in ((a, fa), (b, fb), (b0, fb)):
            _step(gen, cfg, B, f.codes[t], None if f.noise is None else f.noise[t])
    rec = a.export_session(i)
    b.import_session(j, rec if to is None else rec.to(to))
    for t in range(fill, steps):
        codes_b, noise_b = fb.codes[t].clone(), None if fb.noise is None else fb.noise[t].clone()
        codes_b[j] = fa.codes[t][i]                       # the moved session's input and noise follow it to row j
        if noise_b is not None:
            noise_b[j] = fa.noise[t][i]
        ra = _step(a, cfg, B, fa.codes[t], None if fa.noise is None else fa.noise[t])
        rb = _step(b, cfg, B, codes_b, noise_b)
        r0 = _step(b0, cfg, B, fb.codes[t], None if fb.noise is None else fb.noise[t])
        _same_row(ra, i, rb, j)
        for r in range(B):
            if r != j:
                _same_row(r0, r, rb, r)
    for gen in (a, b, b0):
        assert gen.error_flags() == 0


# ---- 1. moved sessions continue bit for bit -----------------------------------------------------------------------------
@pytest.mark.parametrize("B", [3, 40])
@pytest.mark.parametrize("layouts", [("contig", "paged"), ("paged", "contig"), ("int8", "int8"), ("e4m3", "e4m3")])
@pytest.mark.parametrize("fill", [1, 5, 12, 19])          # young, just past a page boundary, full, wrapped
@pytest.mark.parametrize("sampling", [False, True])
def test_moved_session_continues_bit_for_bit(lms, tiny, B, layouts, fill, sampling):
    cfg, _ = tiny
    _move_and_compare(*lms, cfg, B, layouts[0], layouts[1], fill, sampling, i=0, j=B - 1)


# ---- 2. CFG and condition_sum: both model rows travel ---------------------------------------------------------------------
@pytest.mark.parametrize("fill", [5, 19])
@pytest.mark.parametrize("layouts", [("contig", "paged"), ("paged", "contig")])
def test_moved_session_under_cfg(lms, tiny, fill, layouts):
    cfg, _ = tiny
    B = 3
    _move_and_compare(*lms, cfg, B, layouts[0], layouts[1], fill, False, i=1, j=0,
                      extra={"cfg_coef": 2.5, "until": [3, 7, 4]})


@pytest.mark.parametrize("cfg_coef", [1.0, 2.5])
def test_moved_session_with_condition_sum(lms, tiny, cfg_coef):
    """condition_sum rows set through the C ABI (one distinct row per model row on each handle)."""
    L = _lib()
    cfg, _ = tiny
    B, fill, i, j = 3, 6, 2, 0
    MB = 2 * B if cfg_coef != 1.0 else B
    gens = [_gen(m, B, False, "contig", cfg_coef=cfg_coef) for m in lms]
    a, b, b0 = gens
    g = torch.Generator(device="cuda").manual_seed(3)
    cs_a = (0.1 * torch.randn(MB, cfg.dim, generator=g, device="cuda")).to(torch.bfloat16)
    cs_b = (0.1 * torch.randn(MB, cfg.dim, generator=g, device="cuda")).to(torch.bfloat16)
    for gen, cs in ((a, cs_a), (b, cs_b), (b0, cs_b)):
        L.check(gen._lib.b200_lm_set_condition_sum(gen._h, L.ptr(cs), MB))
    fa, fb = Feed(cfg, a, B, fill + STEPS_AFTER, False, 1), Feed(cfg, b, B, fill + STEPS_AFTER, False, 2)
    for t in range(fill):
        for gen, f in ((a, fa), (b, fb), (b0, fb)):
            _step(gen, cfg, B, f.codes[t], None)
    b.import_session(j, a.export_session(i))
    for t in range(fill, fill + STEPS_AFTER):
        codes_b = fb.codes[t].clone()
        codes_b[j] = fa.codes[t][i]
        ra, rb, r0 = _step(a, cfg, B, fa.codes[t], None), _step(b, cfg, B, codes_b, None), _step(b0, cfg, B, fb.codes[t], None)
        _same_row(ra, i, rb, j)
        for r in range(B):
            if r != j:
                _same_row(r0, r, rb, r)
    # condition_sum on one side only is refused
    rec = a.export_session(i)
    b0._stop()
    plain = _gen(lms[2], B, False, "contig", cfg_coef=cfg_coef)
    with pytest.raises(ValueError):
        plain.import_session(0, rec)


# ---- 3. different batch sizes ---------------------------------------------------------------------------------------------
def test_moved_session_into_another_batch_size(lms, tiny):
    """B=3 -> B=40 changes the GEMM and attention plans: logits within |d| <= 0.08, greedy flips only where the top-2 gap
    allows."""
    cfg, _ = tiny
    fill, i, j = 12, 1, 27
    a, b = _gen(lms[0], 3, False), _gen(lms[1], 40, False)
    fa, fb = Feed(cfg, a, 3, fill + STEPS_AFTER, False, 1), Feed(cfg, b, 40, fill + STEPS_AFTER, False, 2)
    for t in range(fill):
        _step(a, cfg, 3, fa.codes[t], None)
        _step(b, cfg, 40, fb.codes[t], None)
    b.import_session(j, a.export_session(i))
    worst, flips = 0.0, 0
    for t in range(fill, fill + STEPS_AFTER):
        codes_b = fb.codes[t].clone()
        codes_b[j] = fa.codes[t][i]
        ra, rb = _step(a, cfg, 3, fa.codes[t], None), _step(b, cfg, 40, codes_b, None)
        dep_a = a.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, 3, cfg.card)).cpu()
        worst = max(worst, (ra[0][i].float() - rb[0][j].float()).abs().max().item())
        _, unexcused = greedy_unexcused(rb[1][:, j], ra[1][:, i], dep_a[:, i], 0.08)
        _, u = greedy_unexcused(rb[2][j, :1], ra[2][i, :1], ra[0][i:i + 1], 0.08)
        flips += unexcused + u
        if not (torch.equal(ra[2][i], rb[2][j]) and torch.equal(ra[1][:, i], rb[1][:, j])):
            break                     # after an excused flip the two sessions' histories differ
    assert worst <= 0.08, worst
    assert flips == 0


# ---- 4. round trip --------------------------------------------------------------------------------------------------------
def _flat_state(gen):
    out = {}
    for mod, st in gen.get_streaming_state().items():
        for k, v in vars(st).items():
            if isinstance(v, torch.Tensor):
                out[f"{mod}.{k}"] = v.clone()
            elif isinstance(v, __import__("types").SimpleNamespace):
                for k2, v2 in vars(v).items():
                    if isinstance(v2, torch.Tensor):
                        out[f"{mod}.{k}.{k2}"] = v2.clone()
    return out


def _assert_state_equal(x, y):
    assert x.keys() == y.keys()
    for k in x:
        assert torch.equal(x[k].view(torch.uint8) if x[k].dtype == torch.bfloat16 else x[k],
                           y[k].view(torch.uint8) if y[k].dtype == torch.bfloat16 else y[k]), k


@pytest.mark.parametrize("layout", ["contig", "paged", "int8"])
@pytest.mark.parametrize("fill", [5, 19])
def test_round_trip_restores_the_state(lms, tiny, layout, fill):
    cfg, _ = tiny
    B, r = 3, 1
    gen = _gen(lms[0], B, True, layout)
    f = Feed(cfg, gen, B, fill, True, 4)
    for t in range(fill):
        _step(gen, cfg, B, f.codes[t], f.noise[t])
    before, usage = _flat_state(gen), gen.kv_pool_usage()
    rec = gen.export_session(r)
    m = torch.zeros(B, dtype=torch.bool)
    m[r] = True
    gen.reset_streaming(m)
    if layout == "paged":
        assert gen.kv_pool_usage()[0] < usage[0]
    gen.import_session(r, rec)
    _assert_state_equal(before, _flat_state(gen))      # offset_cpu (a host integer, zeroed by the reset) is not compared
    assert gen.kv_pool_usage() == usage


# ---- 5. size ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["contig", "paged", "int8"])
def test_record_size_follows_the_fill(lms, tiny, layout):
    cfg, _ = tiny
    B = 3
    gen = _gen(lms[0], B, False, layout)
    Kc, CT = cfg.n_q + 1, max(cfg.delays) + 2
    c16 = lambda n: -(-n // 16) * 16
    kv_off = -(-(256 + c16(1) + c16(8 * Kc * CT) + c16(8) + c16(8)) // 256) * 256
    slot = cfg.num_layers * 2 * cfg.num_heads * (132 if layout == "int8" else 256)
    f = Feed(cfg, gen, B, 19, False, 5)
    done = 0
    for fill in (0, 1, 4, 12, 19):                     # empty, one slot, a page boundary, full, wrapped
        while done < fill:
            _step(gen, cfg, B, f.codes[done], None)
            done += 1
        rec = gen.export_session(2)
        assert rec.numel() == kv_off + slot * min(fill, cfg.context), fill


# ---- 6. rejections change nothing ------------------------------------------------------------------------------------------
def _stepped(lm, cfg, B, steps, seed, **kw):
    gen = _gen(lm, B, False, **kw)
    f = Feed(cfg, gen, B, steps, False, seed)
    for t in range(steps):
        _step(gen, cfg, B, f.codes[t], None)
    return gen


def _refused(dst, row, rec, exc, code=None):
    state, usage = _flat_state(dst), dst.kv_pool_usage()
    with pytest.raises(exc) as e:
        dst.import_session(row, rec)
    if code is not None:
        assert e.value.code == code
    _assert_state_equal(state, _flat_state(dst))
    assert dst.kv_pool_usage() == usage


def _record(lm, cfg, B, steps, seed, **kw):
    gen = _stepped(lm, cfg, B, steps, seed, **kw)
    rec = gen.export_session(0)
    _LIVE.remove(gen)
    gen._stop()
    return rec


def _stop(gen):
    _LIVE.remove(gen)
    gen._stop()


def test_rejections_change_nothing(lms, tiny):
    from moshi_b200.models import LMModel
    L = _lib()
    cfg, _ = tiny
    B = 3
    src, dst_lm, twin_lm = lms
    rec12, rec19 = _record(src, cfg, B, 12, 1), _record(src, cfg, B, 19, 2)
    # a pool with too few free pages: 4 pages of 4 slots, each row holds one, the record needs three
    dry = _stepped(dst_lm, cfg, B, 4, 3, pool=16, page=4)
    assert dry.kv_pool_usage() == (3, 4)
    _refused(dry, 0, rec12, L.B200Error, L.B200_ERR_STATE)
    _stop(dry)
    short = _stepped(dst_lm, cfg, B, 4, 4, capacity=8)
    _refused(short, 1, rec12, L.B200Error, L.B200_ERR_STATE)     # a short ring smaller than the fill
    _refused(short, 1, rec19, L.B200Error, L.B200_ERR_STATE)     # a wrapped session sent to a short ring
    _stop(short)
    # exporting a short-ring row that stepped past its capacity
    over = _stepped(src, cfg, B, 10, 5, capacity=8)
    assert over.error_flags() == 4
    with pytest.raises(L.B200Error) as e:
        over.export_session(0)
    assert e.value.code == L.B200_ERR_STATE
    _stop(over)
    # another model configuration, another storage type, CFG on one side only
    other_cfg = tiny_lm_config(num_layers=2)
    other = LMModel(other_cfg, synth_lm_state_dict(other_cfg, seed=1), device="cuda")
    refused = [_record(other, cfg, B, 3, 7), _record(src, cfg, B, 3, 8, layout="int8"), _record(src, cfg, B, 3, 9, cfg_coef=2.0)]
    dst = _stepped(dst_lm, cfg, B, 6, 6)
    for rec in refused:
        _refused(dst, 0, rec, ValueError)
    # a truncated record, a bad magic, a row out of range
    _refused(dst, 0, rec12[:-16], AssertionError)
    bad = rec12.clone()
    bad[0] ^= 1
    _refused(dst, 0, bad, ValueError)
    _refused(dst, B, rec12, ValueError)
    _refused(dst, -1, rec12, ValueError)
    with pytest.raises(ValueError):
        dst.export_session(B)
    # after all that, the destination still steps as its twin
    twin = _stepped(twin_lm, cfg, B, 6, 6)
    f = Feed(cfg, dst, B, 3, False, 10)
    for t in range(3):
        x, y = _step(dst, cfg, B, f.codes[t], None), _step(twin, cfg, B, f.codes[t], None)
        for r in range(B):
            _same_row(x, r, y, r)


# ---- 7. Mimi ----------------------------------------------------------------------------------------------------------------
def test_mimi_session_moves_bit_for_bit(lms):
    from moshi_b200.models import MimiModel
    msd = synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED)
    m1, m2 = MimiModel(MimiConfig(), msd, device="cuda"), MimiModel(MimiConfig(), msd, device="cuda")
    B, K = 3, m1.num_codebooks
    m1.streaming_forever(B)
    m2.streaming_forever(B)
    g = torch.Generator().manual_seed(11)
    pcm1, pcm2 = 0.1 * torch.randn(8, B, 1, 1920, generator=g), 0.1 * torch.randn(8, B, 1, 1920, generator=g)
    codes1, codes2 = torch.randint(0, 2048, (8, B, K, 1), generator=g), torch.randint(0, 2048, (8, B, K, 1), generator=g)
    for t in range(4):
        for m, p, c in ((m1, pcm1, codes1), (m2, pcm2, codes2)):
            m.encode(p[t].cuda())
            m.decode(c[t].cuda())
    rec = m1.export_session(0)
    m2.import_session(2, rec)
    for t in range(4, 8):
        p2, c2 = pcm2[t].clone(), codes2[t].clone()
        p2[2], c2[2] = pcm1[t][0], codes1[t][0]
        e1, e2 = m1.encode(pcm1[t].cuda()), m2.encode(p2.cuda())
        d1, d2 = m1.decode(codes1[t].cuda()), m2.decode(c2.cuda())
        assert torch.equal(e1[0], e2[2]), t
        assert torch.equal(d1[0], d2[2]), t
    # an LM record into Mimi and the reverse
    gen = _gen(lms[0], B, False)
    with pytest.raises(ValueError):
        m2.import_session(0, gen.export_session(0))
    with pytest.raises(ValueError):
        gen.import_session(0, rec)
    with pytest.raises(AssertionError):
        m2.import_session(0, rec[:-16])
    m1._stop()
    m2._stop()


# ---- 8. DialogueService ------------------------------------------------------------------------------------------------------
def _service_models():
    from moshi_b200.models import LMModel, MimiModel
    cfg = tiny_lm_config(card=2048)
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    msd = synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED)
    return cfg, LMModel(cfg, sd, device="cuda"), MimiModel(MimiConfig(), msd, device="cuda")


def test_service_session_moves_mid_stream():
    from moshi_b200.serving import DialogueService
    B, frames, move_at = 3, 14, 6
    cfg, lm_a, mimi_a = _service_models()
    _, lm_b, mimi_b = _service_models()
    _, lm_r, mimi_r = _service_models()
    pool = B * 64                                            # one page of the default 64 slots per slot
    src = DialogueService(B, lm_a, mimi_a, use_sampling=False, kv_pool_frames=pool)
    dst = DialogueService(B, lm_b, mimi_b, use_sampling=False)
    ref = DialogueService(B, lm_r, mimi_r, use_sampling=False, kv_pool_frames=pool)
    try:
        _service_move(cfg, B, frames, move_at, src, dst, ref)
    finally:
        for svc in (src, dst, ref):
            svc.close()


def _service_move(cfg, B, frames, move_at, src, dst, ref):
    from moshi_b200.serving import ACTIVE
    g = torch.Generator().manual_seed(12)
    pcm_a = (0.1 * torch.randn(frames, B, 1920, generator=g)).numpy()
    pcm_b = (0.1 * torch.randn(frames, B, 1920, generator=g)).numpy()

    def run(svc, pcm):
        out = np.zeros((B, 1920), dtype=np.float32)
        tok = np.zeros((B, cfg.dep_q + 1), dtype=np.int64)
        flags = np.zeros(B, dtype=np.uint8)
        svc.step(np.ascontiguousarray(pcm.reshape(-1)), out, tok, updates=[ACTIVE] * B, flags_out=flags)
        return out, tok, flags

    for t in range(move_at):
        run(src, pcm_a[t])
        run(ref, pcm_a[t])
        run(dst, pcm_b[t])
    used = src.lm_gen.kv_pool_usage()[0]
    dst.import_session(2, src.export_session(1))
    src.release([1])
    assert src.lm_gen.kv_pool_usage()[0] == used - 1         # the slot's one 64-slot page
    for t in range(move_at, frames):
        p = pcm_b[t].copy()
        p[2] = pcm_a[t][1]
        o_r, t_r, f_r = run(ref, pcm_a[t])
        o_b, t_b, f_b = run(dst, p)
        assert f_b[2] == f_r[1] and np.array_equal(t_b[2], t_r[1]) and np.array_equal(o_b[2], o_r[1]), t


# ---- 9. across GPUs ------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("sampling", [False, True])
def test_moved_session_across_gpus(lms, tiny, sampling):
    from moshi_b200.models import LMModel
    cfg, sd = tiny
    lm1, lm1_twin = LMModel(cfg, sd, device="cuda:1"), LMModel(cfg, sd, device="cuda:1")
    _move_and_compare(lms[0], lm1, lm1_twin, cfg, 3, "contig", "paged", 5, sampling, i=0, j=2, to="cuda:1")
