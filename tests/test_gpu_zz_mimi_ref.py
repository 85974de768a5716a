"""GPU: Mimi's kernels against the fp64 reference (tests/util.py MimiRef64), stage by stage, at serving batch and across the
wrap of the bottleneck transformers' 250-slot rings.

Every SEANet module, both transformers (each layer's new ring entries and the output), the down-sampling conv, the RVQ codes,
the dequantised and up-sampled latents and the PCM are judged against float64, teacher-forced on the device's own taps, under
|got - want| <= 2^-20 |want| + c rms with the constants MIMI_C_TC of tests/util.py (the fp32 oracle's constants, widened for
the 3xTF32 kernels where measured).  The reference uses the kernels' fp32 RoPE frequencies (device_rope_freqs).

The reference runs on selected rows only: row 0, the last row, the rows on each side of every 64-session tile edge (the tile
of the layers with two steps per session; the 4- and 8-session tiles of the deeper SEANet layers are covered at rows 3 / 4 and
7 / 8) and the first row of the last 4-, 8- and 64-session group.  Its host cost is a few hundredths of a second per row and
frame for encode and decode together.  On one H100 80GB HBM3 (power limit 700 W) the whole file ran in 149 s, 118 s of it
the 61 batches of test_every_stage_matches_fp64_at_serving_batch; worst ratio 0.95 (encoder taps, B = 89).
"""
import ctypes as C
import time

import pytest
import torch

from moshi_b200 import _lib
from moshi_b200.config import MimiConfig
from moshi_b200.synth import synth_mimi_state_dict
from oracle import scenarios
from tests.util import (MIMI_C_TC, MimiRef64, attn_mask64, device_rope_freqs, cptr, mimi_checkpoints, mimi_kind, mimi_plan_batches,
                        mimi_ratios, mimi_tc_chain_factor, ring_attention64, rope64, rvq_unexcused, RVQ_GAP_BOUND)

pytestmark = pytest.mark.gpu

CFG = MimiConfig()
TRS = ("encoder_transformer", "decoder_transformer")
LAST_DEC = "dec.14"
TOKEN_MAJOR = ("enc.14", "enc.tr", "dec.up", "dec.tr")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- op level: one ring attention step ---------------------------------------------------------------------------------------
RING_C = 2.0 ** -17


def test_ring_attn_step_matches_fp64_across_the_wrap():
    """b200_op_mimi_ring_attn (H 8, T 2, cap = context = 250) at offsets on both sides of the fill and the wrap and one hour
    into a stream, executing and paused.  Needle keys (score about +10 for both queries) sit on the oldest in-context key, on
    the two slots the step overwrites (an executing row must not see their old keys, a paused row attends to them) and on slots
    0 and cap - 1.  With T = 2, query 0 of a wrapped step sees 249 keys: its oldest key was just overwritten by query 1's."""
    lib = _lib.lib()
    H, D, T, cap = 8, 64, 2, 250
    offs = [0, 1, 2, 124, 248, 249, 250, 251, 252, 499, 500, 45000]
    paused = [0, 124, 249, 250, 45000]
    off = torch.tensor(offs + paused)
    ex = torch.tensor([True] * len(offs) + [False] * len(paused))
    B = len(off)
    g = torch.Generator().manual_seed(17)
    qkv = torch.randn(B, T, 3, H, D, generator=g)
    pos = off[:, None] + torch.arange(T)[None]
    fr = device_rope_freqs(D, CFG.tr_max_period)
    q = rope64(qkv[:, :, 0].double(), pos, CFG.tr_max_period, fr)
    k_new = rope64(qkv[:, :, 1].double(), pos, CFG.tr_max_period, fr)
    kr = torch.full((B, H, cap, D), float("nan"))
    vr = torch.full((B, H, cap, D), float("nan"))
    needle = (80.0 * (q[:, 0] / q[:, 0].pow(2).sum(-1, keepdim=True) + q[:, 1] / q[:, 1].pow(2).sum(-1, keepdim=True))).float()
    for b in range(B):
        o = int(off[b])
        n = min(o, cap)
        kr[b, :, :n] = torch.randn(H, n, D, generator=g)
        vr[b, :, :n] = torch.randn(H, n, D, generator=g)
        slots = {0, cap - 1, o % cap, (o + 1) % cap, (o + 1 - 249) % cap}
        for s in slots:
            if s < n:
                kr[b, :, s] = needle[b]
                vr[b, :, s] = 4 * torch.randn(H, D, generator=g)
    allowed = attn_mask64(off, T, cap, cap, ex)
    kw, vw = kr.double().clone(), vr.double().clone()
    for b in range(B):
        if ex[b]:
            for t in range(T):
                kw[b, :, int(pos[b, t]) % cap] = k_new[b, t]
                vw[b, :, int(pos[b, t]) % cap] = qkv[b, t, 2].double()
    want = ring_attention64(q, kw, vw, allowed)                                          # [B, T, H, D]
    assert int(allowed[6, 0].sum()) == 249 and int(allowed[6, 1].sum()) == 250          # offset 250: query 0 sees 249 keys

    d_qkv = qkv.reshape(B, T, 3 * H * D).contiguous().cuda()
    d_k, d_v = kr.cuda(), vr.cuda()
    hi = torch.full((B, T, H * D), float("nan"), device="cuda")
    lo = torch.full_like(hi, float("nan"))
    d_off, d_ex = off.cuda(), ex.to(torch.uint8).cuda()
    _lib.check(lib.b200_op_mimi_ring_attn(cptr(d_qkv), cptr(d_k), cptr(d_v), cptr(hi), cptr(lo), cptr(d_off), cptr(d_ex), B, H, T, cap, cap,
                                          C.c_float(CFG.tr_max_period), _stream()))
    torch.cuda.synchronize()
    got = (hi.double() + lo.double()).cpu().view(B, T, H, D)
    r = mimi_ratios(got.reshape(B * T * H, D), want.reshape(B * T * H, D), RING_C).view(B, T, H)
    worst = r.amax(dim=(1, 2))
    print("ring attention worst ratio per row: " + ", ".join(f"{o}{'' if e else 'p'}: {float(x):.3f}" for o, e, x in zip(off.tolist(), ex.tolist(), worst)))
    # the rings: untouched slots bit for bit, v copied bit for bit, k within fp32 rounding of the fp64 rotation of the fp32 angle
    gk, gv = d_k.cpu(), d_v.cpu()
    for b in range(B):
        written = {int(pos[b, t]) % cap for t in range(T)} if ex[b] else set()
        keep = [s for s in range(cap) if s not in written]
        assert torch.equal(gk[b][:, keep].view(torch.int32), kr[b][:, keep].view(torch.int32)), b
        assert torch.equal(gv[b][:, keep].view(torch.int32), vr[b][:, keep].view(torch.int32)), b
        for t in range(T if ex[b] else 0):
            s = int(pos[b, t]) % cap
            assert torch.equal(gv[b, :, s], qkv[b, t, 2]), (b, t)
            raw = qkv[b, t, 1].double()
            mag = raw.view(H, D // 2, 2).abs().sum(-1).repeat_interleave(2, -1)
            err = (gk[b, :, s].double() - k_new[b, t]).abs()
            assert (err <= 2.0 ** -21 * mag).all(), (int(off[b]), t, float((err / mag).max()))
    assert (worst <= 1).all(), worst
    # refusals: T > 4, or the scores of T queries over the ring above 48 KB of shared memory.  The buffers are sized for each
    # requested shape, so the call is in bounds whatever it does.
    for Tb, capb in ((5, 250), (2, 6100), (4, 3100)):
        assert (Tb * 64 + Tb * capb) * 4 > 48 * 1024 or Tb > 4
        q1 = torch.zeros(1, Tb, 3 * 64, device="cuda")
        k1, v1 = torch.zeros(1, 1, capb, 64, device="cuda"), torch.zeros(1, 1, capb, 64, device="cuda")
        o1, o2 = torch.zeros(1, Tb, 64, device="cuda"), torch.zeros(1, Tb, 64, device="cuda")
        rc = lib.b200_op_mimi_ring_attn(cptr(q1), cptr(k1), cptr(v1), cptr(o1), cptr(o2), cptr(d_off[:1]), cptr(d_ex[:1]), 1, 1, Tb, capb,
                                        capb, C.c_float(CFG.tr_max_period), _stream())
        assert rc == _lib.B200_ERR_SHAPE, (Tb, capb, rc)


# ---- handle level ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd():
    return synth_mimi_state_dict(CFG, seed=scenarios.MIMI_SEED)


@pytest.fixture(scope="module")
def gpu(sd):
    from moshi_b200.models import MimiModel
    return MimiModel(CFG, sd, device="cuda")


def select_rows(B: int, extra: tuple[int, ...] = ()) -> list[int]:
    """Row 0, the last row, the rows on each side of the 4-, 8- and 64-session tile edges, the first row of the last 4-, 8- and
    64-session group (it sits in the partial last tile), and ``extra`` (rows a case acts on)."""
    rows = {0, B - 1} | {r for r in (3, 4, 7, 8) if r < B} | {(B - 1) // g * g for g in (4, 8, 64)} | set(extra)
    for m in range(64, B, 64):
        rows |= {m - 1, m}
    return sorted(rows)


def _read_state(gpu, name: str, shape, dtype=torch.float32) -> torch.Tensor:
    t = torch.empty(shape, dtype=dtype, device="cuda")
    _lib.check(gpu._lib.b200_mimi_state_read(gpu._h, name.encode(), _lib.ptr(t), t.numel() * t.element_size()))
    return t


def _write_state(gpu, name: str, t: torch.Tensor) -> None:
    t = t.contiguous().cuda()
    _lib.check(gpu._lib.b200_mimi_state_write(gpu._h, name.encode(), _lib.ptr(t), t.numel() * t.element_size()))


def _rings(gpu, B: int, rows: list[int]) -> dict:
    """Both transformers' rings of the selected rows: {"<which>.<l>.k" / ".v": [R, H, cap, 64]}."""
    H, cap = CFG.tr_num_heads, CFG.tr_context
    idx = torch.tensor(rows, device="cuda")
    out = {}
    for which in TRS:
        for l in range(CFG.tr_num_layers):
            for kv in ("k", "v"):
                out[f"{which}.{l}.{kv}"] = _read_state(gpu, f"{which}.layers.{l}.{kv}", (B, H, cap, 64))[idx].cpu()
    return out


def _offsets(gpu, B: int, rows: list[int]) -> dict:
    return {w: _read_state(gpu, w + ".offset", (B,), torch.int64).cpu()[rows] for w in TRS}


def _taps(gpu, names: list[str], B: int, rows: list[int]) -> dict:
    out = {}
    for n in names:
        try:
            t = gpu.debug_buffer(n)
        except ValueError:
            continue
        if n in ("enc.latent", "dec.latent"):
            out[n] = t.view(B, -1, 1)[rows].cpu()
        elif n in TOKEN_MAJOR:
            out[n] = t.view(B, -1, CFG.dimension)[rows].transpose(1, 2).cpu()
        else:
            out[n] = t.view(B, _channels(n), -1)[rows].cpu()
    return out


def _channels(tap: str) -> int:
    from moshi_b200.synth import seanet_layout
    side, idx = tap.split(".")
    for kind, i, cin, cout, *_ in seanet_layout(CFG)[0 if side == "enc" else 1]:
        if i == int(idx):
            return cout
    raise KeyError(tap)


def _tap_names():
    from moshi_b200.synth import seanet_layout
    enc, dec = seanet_layout(CFG)
    return [f"enc.{l[1]}" for l in enc] + ["enc.tr", "enc.latent"], ["dec.latent", "dec.up", "dec.tr"] + [f"dec.{l[1]}" for l in dec]


class Verdict:
    """Worst ratio per checkpoint kind and the first failure, in frame order."""

    def __init__(self, case: str):
        self.case, self.worst, self.first = case, {}, None

    def add(self, frame: int, rows: list[int], name: str, r: torch.Tensor, row_ids=None):
        kind = "codes" if name == "codes" else mimi_kind(name, LAST_DEC)
        self.worst[kind] = max(self.worst.get(kind, 0.0), float(r.max()) if r.numel() else 0.0)
        bad = (r > 1).nonzero().flatten()
        if len(bad) and self.first is None:
            row = (row_ids if row_ids is not None else rows)[int(bad[0])]
            stage = "rvq" if name == "codes" else name.split(".")[0]
            layer = name.split(".")[1] if name.endswith((".k", ".v")) else None
            self.first = f"frame {frame}, row {row}, stage {stage}, layer {layer}, checkpoint {name}: ratio {float(r[bad[0]]):.3g}"

    def report(self) -> str:
        return f"{self.case}: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(self.worst.items()))


WRAP_OFFSETS = (246, 249, 250, 45000)


def run_case(gpu, sd, B: int, frames: int, *, seed: int = 0, ncb: int = 8, wrap_at: int | None = None, events=None,
             event_rows: tuple[int, ...] = ()) -> Verdict:
    """Streams ``frames`` frames of B sessions through encode and decode and judges the selected rows at every checkpoint.
    ``wrap_at``: before that frame both transformers' rings are refilled with random entries of the stream's magnitude and the
    offsets set to 246 (no wrap), 249 (this step writes slots 249 and 0), 250 (wrapped) and 45 000; the selected rows take the
    four values in turn, so each is judged.  ``events(frame)`` -> (exec_mask [B] or None, reset_mask [B] or None); every row an
    event touches must be in ``event_rows``, which are judged with the selected rows."""
    rows = select_rows(B, event_rows)
    R = len(rows)
    ref = MimiRef64(sd, CFG, R, rope_freqs=device_rope_freqs(64, CFG.tr_max_period))
    enc_names, dec_names = _tap_names()
    pcm = scenarios.mimi_noise(B, frames, seed=seed)
    v = Verdict(f"B={B} ncb={ncb}" + (" wrap" if wrap_at is not None else "") + (" events" if events else ""))
    g = torch.Generator().manual_seed(seed + 1)
    H, cap = CFG.tr_num_heads, CFG.tr_context
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    consts = dict(MIMI_C_TC)
    for kind, side in (("enc", "encoder"), ("dec", "decoder")):
        consts[kind] *= mimi_tc_chain_factor(_lib.lib(), sms, B, side)
    with gpu.streaming(B):
        gpu.set_num_codebooks(ncb)
        for f in range(frames):
            if events is not None:
                ex, rs = events(f)
                for m, full in ((ex, True), (rs, False)):
                    if m is not None:
                        touched = set((m != full).nonzero().flatten().tolist())
                        assert touched <= set(rows), (f, touched - set(rows))
                if rs is not None:
                    gpu.reset_streaming(rs)
                    ref.reset(rs[rows])
                if ex is not None:
                    gpu.set_exec_mask(ex)
                    ref.exec = ex[rows].clone()
            if f == wrap_at:
                pattern = torch.tensor(WRAP_OFFSETS)
                off = pattern.repeat(B)[:B]
                for i, r in enumerate(rows):
                    off[r] = pattern[i % len(pattern)]
                assert B < len(pattern) or set(off[rows].tolist()) == set(WRAP_OFFSETS)
                for which in TRS:
                    _write_state(gpu, which + ".offset", off)
                    ref.offset[which] = off[rows].clone()
                    for l in range(CFG.tr_num_layers):
                        for kv in ("k", "v"):
                            cur = _read_state(gpu, f"{which}.layers.{l}.{kv}", (B, H, cap, 64))
                            scale = cur[:, :, :2 * wrap_at].pow(2).mean().sqrt().item()
                            _write_state(gpu, f"{which}.layers.{l}.{kv}", torch.randn(B, H, cap, 64, generator=g) * scale)
            executing = ref.exec.clone()
            before = _rings(gpu, B, rows)
            off_before = _offsets(gpu, B, rows)
            assert all(torch.equal(off_before[w], ref.offset[w]) for w in TRS), (f, off_before, ref.offset)
            x = pcm[..., f * 1920:(f + 1) * 1920]
            codes = gpu.encode(x.cuda())
            taps = _taps(gpu, enc_names, B, rows)
            enc_rings = [(before[f"{TRS[0]}.{l}.k"], before[f"{TRS[0]}.{l}.v"]) for l in range(CFG.tr_num_layers)]
            want = ref.encode_frame(x[rows], taps, enc_rings)
            dev_codes = codes[rows, :, 0].cpu()
            q = ref.quantize(taps["enc.latent"][..., 0], dev_codes)
            out = gpu.decode(codes)
            dtaps = _taps(gpu, dec_names, B, rows)
            dtaps[LAST_DEC] = out[rows].cpu()
            dec_rings = [(before[f"{TRS[1]}.{l}.k"], before[f"{TRS[1]}.{l}.v"]) for l in range(CFG.tr_num_layers)]
            want.update(ref.decode_frame(dev_codes, dtaps, dec_rings))
            after = _rings(gpu, B, rows)
            for name, got, w, per_head in mimi_checkpoints(want, {**taps, **dtaps}, after, off_before, executing, cap):
                r = mimi_ratios(got, w, consts[mimi_kind(name, LAST_DEC)], per_head)
                v.add(f, rows, name, r, [rows[i] for i in executing.nonzero().flatten()] if per_head else None)
            un = rvq_unexcused(dev_codes, q, RVQ_GAP_BOUND)
            v.add(f, rows, "codes", un.any(dim=1).double() * 2)
            for i in (~executing).nonzero().flatten().tolist():           # a paused row's rings do not change
                for name in after:
                    assert torch.equal(after[name][i].view(torch.int32), before[name][i].view(torch.int32)), (f, rows[i], name)
            off_after = _offsets(gpu, B, rows)
            for w in TRS:
                assert torch.equal(off_after[w], ref.offset[w]), (f, w)
    print(v.report())
    return v


BATCHES = [1, 3, 63, 64, 65, 129, 200, 256]


def test_every_stage_matches_fp64_at_serving_batch(gpu, sd):
    """Encode and decode at each batch of BATCHES, frames 0..2, and at the first and last session count of every run of Mimi's
    plan on this device (tests/util.py mimi_plan_batches) not among them, frames 0 and 1.  Frame 0 takes the replicate-padding
    and zero-carry paths, frame 1 the carried ones.  This is where the fused epilogues the op-level tests cannot reach are
    judged at every plan: GELU, the layer-scaled residual and the consumer's hi / lo split with ELU, in both the kernel's
    2-wide fragment store and the split-K reduction's 4-wide store."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    runs = [(B, 3) for B in BATCHES] + [(B, 2) for B in mimi_plan_batches(_lib.lib(), sms) if B not in BATCHES]
    t0 = time.time()
    verdicts = [run_case(gpu, sd, B, frames, seed=B) for B, frames in runs]
    print(f"{len(runs)} batches in {time.time() - t0:.1f} s")
    fails = [f"{v.case}: {v.first}" for v in verdicts if v.first]
    assert not fails, "\n".join(fails)


def test_ring_wrap_paused_and_reset_rows(gpu, sd):
    """Across the ring wrap without warm-up (two frames, then the rings refilled and the offsets set to 246, 249, 250 and 45 000,
    then three frames), and mid-stream events at 65 sessions: row 5 paused on frames 2 and 3, row 9 reset before frame 3 (its
    next frame goes back through the first-frame paths), row 64 (alone in the second session tile) paused on frame 4."""
    def events(f):
        ex = torch.ones(65, dtype=torch.bool)
        rs = None
        if f in (2, 3):
            ex[5] = False
        if f == 4:
            ex[64] = False
        if f == 3:
            rs = torch.zeros(65, dtype=torch.bool)
            rs[9] = True
        return ex, rs
    verdicts = [run_case(gpu, sd, 65, 5, seed=7, wrap_at=2), run_case(gpu, sd, 65, 5, seed=8, events=events, event_rows=(5, 9, 64)),
                run_case(gpu, sd, 129, 5, seed=9, wrap_at=2)]
    fails = [f"{v.case}: {v.first}" for v in verdicts if v.first]
    assert not fails, "\n".join(fails)


def test_rvq_codebook_counts(gpu, sd):
    """set_num_codebooks at 32 and at 1 (semantic only); 8 is the default of the other cases."""
    verdicts = [run_case(gpu, sd, B, 2, seed=40 + ncb, ncb=ncb) for B, ncb in ((65, 32), (129, 1), (3, 32))]
    fails = [f"{v.case}: {v.first}" for v in verdicts if v.first]
    assert not fails, "\n".join(fails)


def test_rvq_multi_frame_quantize_and_ties_across_chunks(sd):
    """The multi-frame b200_mimi_quantize entry with Q = B * frames not a multiple of 8, at 32 codebooks, on a checkpoint whose
    codebooks hold duplicated centroids at codes 127 / 128 (semantic level 0) and 1023 / 1024 (acoustic level 0): latents that
    land exactly on them tie across the 128-code chunk partials and must resolve to the lower index."""
    from moshi_b200.models import MimiModel
    sd2 = dict(sd)
    for name, a, b in (("rvq_first", 127, 128), ("rvq_rest", 1023, 1024)):
        p = f"quantizer.{name}.vq.layers.0._codebook"
        for key in (".embedding_sum", ".cluster_usage"):
            t = sd2[p + key].clone()
            t[b] = t[a]
            sd2[p + key] = t
    gpu2 = MimiModel(CFG, sd2, device="cuda")
    ref = MimiRef64(sd2, CFG, 1)
    B, frames, K = 3, 5, 32
    Wf = ref.W("quantizer.rvq_first.input_proj.weight")[..., 0]
    Wr = ref.W("quantizer.rvq_rest.input_proj.weight")[..., 0]
    c1 = ref._centroids("quantizer.rvq_first.vq.layers.0._codebook")[127]
    c2 = ref._centroids("quantizer.rvq_rest.vq.layers.0._codebook")[1023]
    tie = torch.linalg.solve(torch.cat([Wf, Wr]), torch.cat([c1, c2]))                  # both projections hit the tied centroids
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(B, CFG.dimension, frames, generator=g) * 0.8
    lat[0, :, 1] = tie.float()
    lat[2, :, 4] = tie.float()
    with gpu2.streaming(B):
        gpu2.set_num_codebooks(K)
        codes = torch.empty(B, K, frames, dtype=torch.int64, device="cuda")
        d_lat = lat.cuda().contiguous()
        _lib.check(gpu2._lib.b200_mimi_quantize(gpu2._h, _lib.ptr(d_lat), frames, _lib.ptr(codes)))
    codes = codes.cpu()
    ref = MimiRef64(sd2, CFG, B * frames)
    flat_lat = lat.permute(0, 2, 1).reshape(B * frames, -1)
    flat_codes = codes.permute(0, 2, 1).reshape(B * frames, K)
    q = ref.quantize(flat_lat, flat_codes)
    un = rvq_unexcused(flat_codes, q, RVQ_GAP_BOUND)
    print(f"multi-frame quantize Q = {B * frames}: {int((flat_codes != q['codes']).sum())} codes differ from fp64, {int(un.sum())} unexcused")
    assert not un.any()
    for b, f in ((0, 1), (2, 4)):
        assert int(codes[b, 0, f]) == 127 and int(codes[b, 1, f]) == 1023, codes[b, :2, f]
