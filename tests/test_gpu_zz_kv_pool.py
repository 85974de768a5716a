"""GPU: paged temporal KV rings (``LMGen.kv_pool_frames``, ``b200_lm_set_kv_pool``).  Paging changes where a key is stored,
not how it is summed, so every comparison with the contiguous ring is bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from moshi_b200.config import LMConfig, MimiConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict, synth_mimi_state_dict
from oracle import scenarios

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    cfg = tiny_lm_config()
    return cfg, synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)


@pytest.fixture(scope="module")
def lm(tiny):
    from moshi_b200.models import LMModel
    cfg, sd = tiny
    return LMModel(cfg, sd, device="cuda")


def _lib():
    from moshi_b200 import _lib
    return _lib


# ---- kernel ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [2, 32])
@pytest.mark.parametrize("cap", [12, 3000])
@pytest.mark.parametrize("page_slots", [4, 16, 64])
@pytest.mark.parametrize("nsplit", [1, 4, 16])
def test_paged_attention_step_equals_contiguous(H, cap, page_slots, nsplit):
    L = _lib()
    lib = L.lib()
    D, B = 128, 5
    g = torch.Generator().manual_seed(H * 7 + cap + page_slots + nsplit)
    # fills: young, last slot before the wrap, past the wrap, a paused row, the first step
    pos = torch.tensor([cap // 3, cap - 1, cap + 7, cap // 2, 0], dtype=torch.int64)
    exec_ = torch.tensor([1, 1, 1, 0, 1], dtype=torch.uint8)
    gd = torch.Generator(device="cuda").manual_seed(int(g.initial_seed()))
    qkv = torch.randn(B, 3 * H * D, generator=gd, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, H, cap, D, generator=gd, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, H, cap, D, generator=gd, device="cuda").to(torch.bfloat16)
    T = -(-cap // page_slots)
    n_pages = B * T + 3
    # a shuffled page permutation; the table maps only the slots the step reads or writes, unmapped pages hold noise
    used = torch.clamp(pos + exec_.long(), max=cap)
    mapped = torch.arange(T)[None, :] * page_slots < used[:, None]
    table = torch.full((B, T), -1, dtype=torch.int32)
    table[mapped] = torch.randperm(n_pages, generator=g)[:int(mapped.sum())].int()
    kp = torch.randn(n_pages, H, page_slots, D, generator=gd, device="cuda").to(torch.bfloat16)
    vp = torch.randn(n_pages, H, page_slots, D, generator=gd, device="cuda").to(torch.bfloat16)
    m, tab = mapped.cuda(), table.cuda().long()
    for ring, pool in ((k, kp), (v, vp)):
        pad = torch.zeros(B, H, T * page_slots, D, dtype=torch.bfloat16, device="cuda")
        pad[:, :, :cap] = ring
        pages = pad.view(B, H, T, page_slots, D).permute(0, 2, 1, 3, 4)      # [B][T][H][page_slots][D]
        pool[tab[m]] = pages[m]
    kp0 = kp.clone()
    dev = dict(qkv=qkv, k=k, v=v, kp=kp, vp=vp, table=table.cuda(), pos=pos.cuda(), exec_=exec_.cuda())
    k0 = k.clone()
    out_c = torch.empty(B, H * D, dtype=torch.bfloat16, device="cuda")
    out_p = torch.empty_like(out_c)
    st = L.current_stream(torch.device("cuda"))
    L.check(lib.b200_op_attn_step(L.ptr(dev["qkv"]), L.ptr(dev["k"]), L.ptr(dev["v"]), L.ptr(out_c), L.ptr(dev["pos"]),
                                  L.ptr(dev["exec_"]), B, H, cap, nsplit, 10000.0, st))
    L.check(lib.b200_op_attn_step_paged(L.ptr(dev["qkv"]), L.ptr(dev["kp"]), L.ptr(dev["vp"]), L.ptr(dev["table"]), L.ptr(out_p),
                                        L.ptr(dev["pos"]), L.ptr(dev["exec_"]), B, H, cap, page_slots, nsplit, 10000.0, st))
    torch.cuda.synchronize()
    assert torch.equal(out_p.view(torch.int16), out_c.view(torch.int16))
    for b in range(B):
        s = int(pos[b]) % cap
        pg = int(table[b, s // page_slots])
        if exec_[b]:       # the new key (RoPE'd) and value at the paged address of slot pos % cap
            assert torch.equal(kp[pg, :, s % page_slots].view(torch.int16), k[b, :, s].view(torch.int16)), b
            assert torch.equal(vp[pg, :, s % page_slots].view(torch.int16), v[b, :, s].view(torch.int16)), b
        else:              # a paused row writes nothing
            assert torch.equal(k[b], k0[b]) and (pg < 0 or torch.equal(kp[pg], kp0[pg])), b


@pytest.mark.parametrize("H,cap,nsplit,page_slots", [(32, 3000, 16, 64), (32, 3000, 0, 4), (20, 250, 3, 16), (2, 12, 5, 4)])
def test_paged_attention_step_scenarios_equal_contiguous(H, cap, nsplit, page_slots):
    """The scenarios of test_fused_attention_step (fills at the group and split edges, wraps, paused rows, needles, NaN
    poison past the fill) on paged rings: outputs and every mapped slot bit for bit those of the contiguous kernel.  Needles
    also sit on the last slot of the first page and the first slot of the second, so page boundaries fall on needle keys."""
    from tests.util import attn_scenario
    L = _lib()
    lib = L.lib()
    sc = attn_scenario(H, cap, nsplit, extra_needles=(page_slots - 1, page_slots))
    B, D = sc["B"], 128
    g = torch.Generator().manual_seed(H + cap + page_slots)
    T = -(-cap // page_slots)
    n_pages = B * T + 3
    used = sc["n_valid"]
    mapped = torch.arange(T)[None, :] * page_slots < used[:, None]
    table = torch.full((B, T), -1, dtype=torch.int32)
    table[mapped] = torch.randperm(n_pages, generator=g)[:int(mapped.sum())].int()
    k, v = sc["k"].cuda(), sc["v"].cuda()
    kp = torch.randn(n_pages, H, page_slots, D, generator=g).bfloat16().cuda()
    vp = torch.randn(n_pages, H, page_slots, D, generator=g).bfloat16().cuda()
    m, tab = mapped.cuda(), table.cuda().long()

    def pages(ring):
        pad = torch.zeros(B, H, T * page_slots, D, dtype=torch.bfloat16, device="cuda")
        pad[:, :, :cap] = ring
        return pad.view(B, H, T, page_slots, D).permute(0, 2, 1, 3, 4)       # [B][T][H][page_slots][D]

    kp[tab[m]] = pages(k)[m]
    vp[tab[m]] = pages(v)[m]
    qkv, pos, ex = sc["qkv"].cuda(), sc["pos"].cuda(), sc["mask"].to(torch.uint8).cuda()
    table_d = table.cuda()
    out_c = torch.empty(B, H * D, dtype=torch.bfloat16, device="cuda")
    out_p = torch.empty_like(out_c)
    st = L.current_stream(torch.device("cuda"))
    L.check(lib.b200_op_attn_step(L.ptr(qkv), L.ptr(k), L.ptr(v), L.ptr(out_c), L.ptr(pos), L.ptr(ex), B, H, cap, nsplit, 10000.0, st))
    L.check(lib.b200_op_attn_step_paged(L.ptr(qkv), L.ptr(kp), L.ptr(vp), L.ptr(table_d), L.ptr(out_p), L.ptr(pos), L.ptr(ex), B, H, cap,
                                        page_slots, nsplit, 10000.0, st))
    torch.cuda.synchronize()
    assert torch.isfinite(out_c.float()).all()
    assert torch.equal(out_p.view(torch.int16), out_c.view(torch.int16))
    assert torch.equal(kp[tab[m]].view(torch.int16), pages(k)[m].view(torch.int16))
    assert torch.equal(vp[tab[m]].view(torch.int16), pages(v)[m].view(torch.int16))


# ---- LM step --------------------------------------------------------------------------------------------------------------
def _run(lm, cfg, B, steps, sampling, use_graph, pool=None, page=4, events=None, seed=5):
    """Steps an LMGen (`pool` = kv_pool_frames) and records per step: text logits, audio tokens, output tokens, flags."""
    from moshi_b200.models import LMGen
    gen = LMGen(lm, use_sampling=sampling)
    gen.use_graph = use_graph
    gen.kv_pool_frames, gen.kv_page_slots = pool, page
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, cfg.card, (steps, B, cfg.n_q - cfg.dep_q, 1), generator=g)
    rec = []
    with gen.streaming(B):
        npr = gen._noise_per_row
        noise = torch.empty(steps, B, npr).exponential_(1, generator=g)
        for i in range(steps):
            if events is not None:
                events(gen, i, B)
            out = gen.step(codes[i].cuda(), noise=noise[i].cuda() if sampling else None)
            rec.append((gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).cpu(),
                        gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu(),
                        None if out is None else out.cpu(), gen.error_flags()))
    return rec


def _mask_and_reset_events(gen, i, B):
    scenarios.lm_mask_events(gen, i, B)           # row 1 paused at steps 10-11, reset at step 20
    if i == 31:
        m = torch.zeros(B, dtype=torch.bool)
        m[0] = True
        m[B - 1] = True
        gen.reset_streaming(m)


def _assert_same(a, b, rows=None):
    for i, (x, y) in enumerate(zip(a, b)):
        sel = slice(None) if rows is None else rows
        assert torch.equal(x[0][sel].view(torch.int16), y[0][sel].view(torch.int16)), i
        assert torch.equal(x[1][:, sel], y[1][:, sel]), i
        assert (x[2] is None) == (y[2] is None), i
        if x[2] is not None:
            assert torch.equal(x[2][sel], y[2][sel]), i


@pytest.mark.parametrize("B", [3, 40])
@pytest.mark.parametrize("sampling", [False, True])
@pytest.mark.parametrize("use_graph", [False, True])
def test_paged_lm_step_equals_contiguous(lm, tiny, B, sampling, use_graph):
    """40 steps of a 12-slot ring in pages of 4 (every ring wraps), with paused rows and resets."""
    cfg, _ = tiny
    ref = _run(lm, cfg, B, 40, sampling, use_graph, events=_mask_and_reset_events)
    got = _run(lm, cfg, B, 40, sampling, use_graph, pool=B * cfg.context, events=_mask_and_reset_events)
    assert all(r[3] == 0 for r in got)
    _assert_same(ref, got)


@torch.no_grad()
def test_paged_mid_size_7b_family_across_the_wrap():
    """Head dim 128, context 3000 (not a multiple of the 64-slot page), steps crossing the wrap after assume_fill(2990)."""
    from moshi_b200.models import LMGen, LMModel
    cfg = LMConfig(dim=1024, num_heads=8, num_layers=4, context=3000, text_card=32000, card=2048,
                   depformer_dim=512, depformer_num_heads=8, depformer_dim_feedforward=2112, depformer_num_layers=2)
    lm7 = LMModel(cfg, synth_lm_state_dict(cfg, seed=5, device="cuda"), device="cuda")
    B, steps = 6, 14
    g = torch.Generator().manual_seed(2)
    codes = torch.randint(0, cfg.card, (steps, B, 8, 1), generator=g).cuda()
    noise = torch.empty(steps, B, 25 + 8 * 250).exponential_(1, generator=g).cuda()

    def run(pool):
        gen = LMGen(lm7)
        gen.kv_pool_frames = pool
        outs = []
        with gen.streaming(B):
            gen.assume_fill(2990)
            for i in range(steps):
                o = gen.step(codes[i], noise=noise[i].contiguous())
                outs.append((o[:, :, 0].cpu(), gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).cpu()))
            assert gen.error_flags() & 8 == 0      # assume_fill leaves ungenerated tokens in the token ring: flag 1 is expected
            if pool:
                assert gen.kv_pool_usage() == (B * 47, B * 47)
        return outs

    ref, got = run(None), run(B * 3000)
    for i, ((ta, la), (tb, lb)) in enumerate(zip(ref, got)):
        assert torch.equal(ta, tb), i
        assert torch.equal(la.view(torch.int16), lb.view(torch.int16)), i
    del lm7
    torch.cuda.empty_cache()


# ---- sharing and isolation ------------------------------------------------------------------------------------------------
def _staggered_resets(gen, i, B):
    m = torch.tensor([(i + b) % 6 == 0 for b in range(B)])
    if i > 0 and m.any():
        gen.reset_streaming(m)


def test_pool_smaller_than_full_rings_shared_by_staggered_sessions(lm, tiny):
    """4 rows of 12-slot rings would need 12 pages of 4; each row is reset every 6 steps, so its live fill never needs more than
    2 pages and a pool of 8 serves all of them: no flag, the same results as the contiguous rings."""
    cfg, _ = tiny
    B = 4
    ref = _run(lm, cfg, B, 30, True, True, events=_staggered_resets)
    got = _run(lm, cfg, B, 30, True, True, pool=8 * 4, events=_staggered_resets)
    assert all(r[3] == 0 for r in got)
    _assert_same(ref, got)


@torch.no_grad()
def test_overfilled_pool_flags_the_last_row_and_spares_the_others(lm, tiny):
    """A pool of 7 pages for 4 rows stepping together: at position 4 every row asks for its second page; pages go in row
    order, so rows 0-2 get them and row 3 does not.  Flag 8, step_host returns B200_ERR_STATE, rows 0-2 stay bit-identical
    to the contiguous rings, and row 3's unserved slots read as zeros in its streaming state."""
    from moshi_b200.models import LMGen
    L = _lib()
    cfg, _ = tiny
    B, steps = 4, 8
    g = torch.Generator().manual_seed(8)
    codes = torch.randint(0, cfg.card, (steps, B, 8), generator=g)

    def run(pool):
        gen = LMGen(lm, use_sampling=False)
        gen.kv_pool_frames, gen.kv_page_slots = pool, 4
        rec, failed = [], []
        with gen.streaming(B):
            for i in range(steps):
                out = torch.empty(B, cfg.dep_q + 1, dtype=torch.int64)
                try:
                    gen.step_host(codes[i].contiguous(), None, out)
                except L.B200Error as e:
                    assert e.code == L.B200_ERR_STATE and "KV pool" in str(e)
                    failed.append(i)
                rec.append((out.clone(), gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).cpu()))
            usage = gen.kv_pool_usage()
            k = gen.get_streaming_state()["lm_model.transformer.layers.0.self_attn"].kv_cache.cache[0].cpu()
            gen.reset_streaming(torch.tensor([False, True, False, False]))
            after = gen.kv_pool_usage()
        return rec, failed, usage, after, k

    ref, failed_ref, *_ = run(None)
    got, failed, usage, after, k = run(7 * 4)
    assert failed_ref == [] and failed == [4, 5, 6, 7]
    assert usage == (7, 7) and after == (5, 7)           # row 1's two pages went back to the pool
    for i in range(1, steps):
        assert torch.equal(got[i][0][:3], ref[i][0][:3]), i
        assert torch.equal(got[i][1][:3].view(torch.int16), ref[i][1][:3].view(torch.int16)), i
    assert (k[3, :, 4:] == 0).all() and (k[3, :, :4] != 0).any()
    assert (k[:3, :, 4:8] != 0).any(dim=-1).all()


# ---- streaming state ------------------------------------------------------------------------------------------------------
def _blob(gen):
    lib, L = gen._lib, _lib()
    n = int(lib.b200_lm_state_bytes(gen._h))
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    L.check(lib.b200_lm_get_state(gen._h, L.ptr(buf), n))
    return buf


def _set_blob(gen, buf):
    L = _lib()
    L.check(gen._lib.b200_lm_set_state(gen._h, L.ptr(buf), buf.numel()))


@torch.no_grad()
def test_streaming_state_moves_between_paged_and_contiguous_handles(tiny):
    from moshi_b200.models import LMGen, LMModel
    cfg, sd = tiny
    lm_a, lm_b = LMModel(cfg, sd, device="cuda"), LMModel(cfg, sd, device="cuda")
    B = 3
    g = torch.Generator().manual_seed(4)
    codes = torch.randint(0, cfg.card, (24, B, 8, 1), generator=g).cuda()
    paged, contig = LMGen(lm_a, use_sampling=False), LMGen(lm_b, use_sampling=False)
    paged.kv_pool_frames, paged.kv_page_slots = B * cfg.context, 4
    with paged.streaming(B), contig.streaming(B):
        assert int(paged._lib.b200_lm_state_bytes(paged._h)) == int(contig._lib.b200_lm_state_bytes(contig._h))
        for i in range(7):
            paged.step(codes[i])
        # round trip on the paged handle, entry by entry
        snap = paged.get_streaming_state()
        first = [paged.step(codes[i]).cpu() for i in range(7, 16)]         # crosses the wrap at 12
        paged.set_streaming_state(snap)
        for i, f in zip(range(7, 16), first):
            assert torch.equal(paged.step(codes[i]).cpu(), f), i
        # paged -> contiguous, whole blob: both continue identically
        blob = _blob(paged)
        _set_blob(contig, blob)
        for i in range(16, 20):
            assert torch.equal(paged.step(codes[i]).cpu(), contig.step(codes[i]).cpu()), i
        # contiguous -> paged, entry by entry after a reset of row 1 in the contiguous handle
        contig.reset_streaming(torch.tensor([False, True, False]))
        contig.step(codes[20])
        paged.set_streaming_state(contig.get_streaming_state())
        assert paged.kv_pool_usage() == (3 + 1 + 3, B * 3)
        for i in range(21, 24):
            assert torch.equal(paged.step(codes[i]).cpu(), contig.step(codes[i]).cpu()), i
        # slots at or past a row's fill read as zeros (row 1 is at fill 4, the others are full)
        k = paged.get_streaming_state()["lm_model.transformer.layers.2.self_attn"].kv_cache.cache[0]
        assert (k[1, :, 4:] == 0).all() and (k[1, :, :4] != 0).any() and (k[0] != 0).any(dim=-1).all()


@torch.no_grad()
def test_round_trip_and_snapshot_that_does_not_fit(tiny):
    from moshi_b200.models import LMGen, LMModel
    L = _lib()
    cfg, sd = tiny
    lm_a, lm_b = LMModel(cfg, sd, device="cuda"), LMModel(cfg, sd, device="cuda")
    B = 3
    g = torch.Generator().manual_seed(6)
    codes = torch.randint(0, cfg.card, (12, B, 8, 1), generator=g).cuda()
    small, contig = LMGen(lm_a, use_sampling=False), LMGen(lm_b, use_sampling=False)
    small.kv_pool_frames, small.kv_page_slots = 6 * 4, 4                 # 6 pages: three rows at fill 9 need 9
    with small.streaming(B), contig.streaming(B):
        for i in range(3):
            small.step(codes[i])
        blob = _blob(small)
        first = [small.step(codes[i]).cpu() for i in range(3, 8)]
        assert small.error_flags() == 0
        _set_blob(small, blob)
        assert small.kv_pool_usage() == (3, 6)
        for i, f in zip(range(3, 8), first):
            assert torch.equal(small.step(codes[i]).cpu(), f)
        for i in range(9):
            contig.step(codes[i])
        before = small.kv_pool_usage()
        with pytest.raises(L.B200Error, match="KV pages"):
            _set_blob(small, _blob(contig))
        with pytest.raises(L.B200Error, match="KV pages"):
            small.set_streaming_state(contig.get_streaming_state())
        assert small.kv_pool_usage() == before
        with pytest.raises(L.B200Error, match="KV pages"):
            small.assume_fill(9)


def test_pool_rejects_8_bit_rings_and_short_rings(lm):
    from moshi_b200.models import LMGen
    for attr, value in (("kv_dtype", "fp8_e4m3"), ("kv_capacity", 8)):
        gen = LMGen(lm)
        gen.kv_pool_frames = 64
        setattr(gen, attr, value)
        with pytest.raises(ValueError, match="bf16 rings"):
            gen.streaming(2)
    gen = LMGen(lm)
    gen.kv_pool_frames, gen.kv_page_slots = 64, 48
    with pytest.raises(ValueError, match="power of two"):
        gen.streaming(2)


# ---- service --------------------------------------------------------------------------------------------------------------
def _service(pool):
    from moshi_b200.models import LMModel, MimiModel
    from moshi_b200.serving import DialogueService
    cfg = tiny_lm_config(card=2048)
    lm = LMModel(cfg, synth_lm_state_dict(cfg, seed=scenarios.LM_SEED), device="cuda")
    mimi = MimiModel(MimiConfig(), synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED), device="cuda")
    return cfg, DialogueService(3, lm, mimi, use_sampling=False, kv_pool_frames=pool)


def test_service_release_returns_pages_and_reused_slot_starts_fresh():
    from moshi_b200.serving import ACTIVE, NODATA, RESET
    B, frames = 3, 10
    cfg, paged = _service(B * 64)              # one 64-slot page per 12-slot ring
    _, contig = _service(None)
    g = torch.Generator().manual_seed(12)
    pcm = (0.1 * torch.randn(frames, B * 1920, generator=g)).numpy()
    for i in range(frames):
        updates = [ACTIVE] * B if i == 0 else [9] * B
        if i == 4:
            updates[1] = NODATA                 # session in slot 1 ends ...
        if i == 6:
            updates[1] = RESET                  # ... and a new one takes the slot
        if i == 5:
            before = paged.lm_gen.kv_pool_usage()
            paged.release([1])
            after = paged.lm_gen.kv_pool_usage()
            assert after[0] < before[0] and after[1] == before[1]
        outs = []
        for svc in (paged, contig):
            pcm_out = np.zeros((B, 1920), dtype=np.float32)
            tok = np.zeros((B, cfg.dep_q + 1), dtype=np.int64)
            flags = np.zeros(B, dtype=np.uint8)
            svc.step(pcm[i].copy(), pcm_out, tok, updates=updates, flags_out=flags)
            outs.append((pcm_out, tok, flags))
        (pa, ta, fa), (pb, tb, fb) = outs
        assert np.array_equal(fa, fb) and np.array_equal(pa, pb), i
        ready = fa.astype(bool)
        assert np.array_equal(ta[ready], tb[ready]), i
    paged.close()
    contig.close()
