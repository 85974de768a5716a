"""GPU: the opt-in 8-bit temporal KV rings (one byte per element + one fp32 scale per key row): e4m3 and int8.

This is NOT the reference's numerics (its ring is bf16, transformer.py:196-288); it exists to halve the 1.57 GB a
session's rings take (SURVEY.md 8f item 3).  Two levels:
  * the fused attention step kernel against an fp32 emulation that stores ``e4m3(x * 448/absmax) * absmax/448`` (or
    ``round(x * 127/absmax) * absmax/127``) for the appended key / value row and attends over the dequantised ring: the
    kernel must agree with that to bf16 rounding, and the bytes + scales it wrote must be the emulation's;
  * the LM step against the oracle with the same emulation in its ring, and the *cost* of the option: logit deviation
    of the fp8-ring model from the bf16-ring model on the same token stream (reported and bounded).
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle.transformer import kv_roundtrip
from tests.util import ATTN_C, ATTN_REL, Q8_FP16_C, Q8_WIDE_C, attn_err_ratio, attn_ref64, attn_scenario, cptr, rope_ref

pytestmark = pytest.mark.gpu


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


FMT = {"fp8_e4m3": (1, 448.0), "int8": (2, 127.0)}


def _encode(t, amax, fmt):
    """Row-scaled bytes as the kernel stores them."""
    qmax = FMT[fmt][1]
    inv = torch.where(amax > 0, torch.full_like(amax, qmax) / amax, torch.zeros_like(amax))     # true division, like the kernel
    y = t.float() * inv[..., None]
    if fmt == "fp8_e4m3":
        return y.to(torch.float8_e4m3fn).view(torch.uint8)
    return (torch.round(y).clamp_(-127, 127) + 128).to(torch.uint8)


def _decode(u8, scale, fmt):
    if fmt == "fp8_e4m3":
        return u8.view(torch.float8_e4m3fn).float() * scale[..., None]
    return (u8.float() - 128.0) * scale[..., None]


def _q8_step(sc: dict, fmt: str, nsplit: int, label: str, c: float = ATTN_C + Q8_FP16_C) -> float:
    """One 8-bit step on a scenario of tests.util.attn_scenario: the scenario's bf16 rings are stored in the kernel's format
    (poisoned slots: byte 0x7F, NaN scale) and the outputs are compared with attn_ref64 over the dequantised ring, whose new
    slot is what the kernel wrote (checked against the emulation separately)."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    B, H, cap = sc["B"], sc["H"], sc["cap"]
    kind, qmax = FMT[fmt]
    poison = torch.isnan(sc["k"].float()).any(-1)                                   # [B, H, cap]
    rings = []
    for t in (sc["k"], sc["v"]):
        clean = torch.nan_to_num(t.float()).bfloat16()
        amax = clean.float().abs().amax(-1)
        u8 = _encode(clean, amax, fmt)
        u8[poison] = 0x7F
        scale = torch.where(poison, torch.full_like(amax, float("nan")), amax * (1.0 / qmax))
        rings += [u8.cuda(), scale.cuda()]
    k8, ks, v8, vs = rings
    k8_0, ks_0, v8_0, vs_0 = (r.cpu().clone() for r in rings)
    out = torch.full((B, H * 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    qd, pd, md = sc["qkv"].cuda(), sc["pos"].cuda(), sc["mask"].cuda()
    _lib.check(lib.b200_op_attn_step_q8(cptr(qd), cptr(k8), cptr(v8), cptr(ks), cptr(vs), cptr(out), cptr(pd), cptr(md),
                                        B, H, cap, nsplit, 10000.0, kind, _stream()))
    torch.cuda.synchronize()
    k8, ks, v8, vs = k8.cpu(), ks.cpu(), v8.cpu(), vs.cpu()
    new = torch.zeros(B, H, cap, dtype=torch.bool)
    for b in range(B):
        if sc["mask"][b]:
            new[b, :, int(sc["pos"][b]) % cap] = True
    # every other slot keeps its bytes and scales (poison included)
    assert torch.equal(k8[~new], k8_0[~new]) and torch.equal(v8[~new], v8_0[~new])
    assert torch.equal(ks.view(torch.int32)[~new], ks_0.view(torch.int32)[~new])
    assert torch.equal(vs.view(torch.int32)[~new], vs_0.view(torch.int32)[~new])
    # the appended value is the emulation's exactly; the key within one grid step where sincos moved a bf16 ulp of it
    deq_k, deq_v = _decode(k8, ks, fmt), _decode(v8, vs, fmt)
    rows = sc["mask"]
    v_in = sc["qkv"].view(B, 3, H, 128)[:, 2]
    em_k, em_v = kv_roundtrip(sc["k_rot"][rows], fmt), kv_roundtrip(v_in[rows], fmt)
    got_k = deq_k.permute(0, 2, 1, 3)[new.permute(0, 2, 1)].view(-1, H, 128)
    got_v = deq_v.permute(0, 2, 1, 3)[new.permute(0, 2, 1)].view(-1, H, 128)
    assert torch.equal(got_v, em_v)
    torch.testing.assert_close(got_k, em_k, rtol=0.13, atol=0.05)
    assert (got_k != em_k).float().mean() < 0.02
    want = attn_ref64(sc["q_rot"], deq_k, deq_v, sc["n_valid"])
    ratio = attn_err_ratio(out, want, c=c)
    print(f"{label}: B={B} nsplit={sc['nsplit']}: worst |err| / tolerance {ratio:.3f} "
          f"(tolerance {ATTN_REL:.3g} |want| + {c:.3g} rms)")
    assert torch.isfinite(out.float()).all()
    assert ratio <= 1.0
    return ratio


@pytest.mark.parametrize("fmt", ["int8", "fp8_e4m3"])
@pytest.mark.parametrize("H,cap,nsplit", [(32, 3000, 16), (32, 3000, 0), (20, 250, 5), (2, 12, 3)])
def test_q8_attention_step_matches_emulation(H, cap, nsplit, fmt):
    """The scenarios of the bf16 kernel's test (fills, wraps, paused rows, needles, poison) on the 8-bit rings: the kernel
    agrees with fp64 attention over the dequantised ring within the bf16 rule plus the fp16 budget Q8_FP16_C."""
    _q8_step(attn_scenario(H, cap, nsplit), fmt, nsplit, f"{fmt} attn step H={H} cap={cap}")


@pytest.mark.parametrize("fmt", ["int8", "fp8_e4m3"])
def test_q8_attention_step_query_range(fmt):
    """The supported query range, |q| <= 256 per element of the rotated query: random queries up to that bound over a full
    ring, and the worst case, a query lined up with a key whose every byte is the format's largest (each fp16 lane partial
    then sums four products of 22.6 x 448 = 40544 for e4m3, below the fp16 limit 65504)."""
    sc = attn_scenario(32, 3000, 0, q_scale=85.0, needles=False, seed=2)
    _q8_step(sc, fmt, 0, f"{fmt} attn step, random |q| <= 256", c=ATTN_C + Q8_WIDE_C)
    # worst case: rows at position 0 (no rotation), q = +-256, the new key = sign(q) (every byte at +-qmax)
    B, H, cap = 4, 2, 64
    g = torch.Generator().manual_seed(9)
    sign = torch.randint(0, 2, (B, H, 128), generator=g).float() * 2 - 1
    qkv = torch.cat([sign * 256, sign, torch.randn(B, H, 128, generator=g)], dim=1).reshape(B, 3 * H * 128).bfloat16()
    pos, mask = torch.zeros(B, dtype=torch.int64), torch.ones(B, dtype=torch.bool)
    k = torch.full((B, H, cap, 128), float("nan")).bfloat16()
    q_in, k_in, v_in = (qkv.view(B, 3, H, 128)[:, i] for i in range(3))
    k_ref, v_ref = k.clone(), k.clone()
    k_ref[:, :, 0], v_ref[:, :, 0] = k_in, v_in
    n_valid = torch.ones(B, dtype=torch.int64)
    worst = dict(H=H, cap=cap, B=B, nsplit=1, qkv=qkv, k=k, v=k.clone(), pos=pos, mask=mask, n_valid=n_valid, q_rot=q_in,
                 k_rot=k_in, k_ref=k_ref, v_ref=v_ref)
    _q8_step(worst, fmt, 1, f"{fmt} attn step, q = +-256 lined up with a key at the format's largest bytes")


@pytest.mark.parametrize("fmt,use_graph", [("int8", False), ("int8", True), ("fp8_e4m3", True)])
def test_q8_ring_lm_matches_emulating_oracle(fmt, use_graph):
    """LM steps with an 8-bit ring against the oracle whose ring holds the same rounded rows (teacher-synchronised)."""
    from moshi_b200.config import tiny_lm_config
    from moshi_b200.models import LMGen, LMModel
    from moshi_b200.synth import synth_lm_state_dict
    from oracle import scenarios
    from oracle.lm import LMOracle, LMSpec
    cfg = tiny_lm_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    lm = LMModel(cfg, sd, device="cuda")
    B, steps = scenarios.LM_B, 20
    codes = scenarios.lm_input_codes(cfg, B, steps)
    gen = LMGen(lm, use_sampling=False)
    gen.kv_dtype = fmt
    gen.use_graph = use_graph
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, tie_break="index", kv_quant=fmt)
    orc.streaming(B)
    worst = 0.0
    agree = total = 0
    with gen.streaming(B):
        for i in range(steps):
            dbg = {}
            orc.step(codes[i], None, None, debug=dbg)
            gen.step(codes[i].cuda())
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            worst = max(worst, (tl - dbg["text_logits"].float()[:, 0, 0]).abs().max().item())
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            agree += int((tt == dbg["text_token"]).sum())
            total += B
            pos = (orc.offsets % orc.cache.shape[2])        # keep the oracle on the GPU's token trajectory
            for b in range(B):
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print(f"{fmt} ring LM vs emulating oracle (graph={use_graph}): worst text-logit diff {worst:.3e}, greedy text tokens equal {agree}/{total}")
    assert worst < 0.12
    assert agree / total > 0.9


@pytest.mark.parametrize("fmt,outlier,bound", [("int8", 1.0, 0.02), ("fp8_e4m3", 1.0, 0.05), ("int8", 8.0, 0.08), ("fp8_e4m3", 8.0, 0.06)])
def test_q8_ring_cost_against_exact_ring(fmt, outlier, bound):
    """What the option costs: attention over a full 3000-slot 8-bit ring against fp32 attention over the unquantised
    keys / values (keys with a few large channels, as rotary models have).  Reported as relative RMS error of the head
    outputs; the bf16 ring's own error on the same data is printed beside it."""
    from moshi_b200 import _lib
    lib = _lib.lib()
    kind, qmax = FMT[fmt]
    B, H, cap = 2, 8, 3000
    g = torch.Generator().manual_seed(5)
    Cd = H * 128
    chan = torch.ones(128)
    chan[torch.randperm(128, generator=g)[:6]] = outlier                  # outlier channels
    hist_k = (torch.randn(B, H, cap, 128, generator=g) * chan).bfloat16()
    hist_v = torch.randn(B, H, cap, 128, generator=g).bfloat16()
    qkv = torch.randn(B, 3 * Cd, generator=g).bfloat16()
    pos = torch.full((B,), 2 * cap + 11, dtype=torch.int64)
    mask = torch.ones(B, dtype=torch.bool)
    q_in, k_in, v_in = (qkv[:, j * Cd:(j + 1) * Cd].reshape(B, H, 128) for j in range(3))
    q_rot, k_rot = rope_ref(q_in, pos), rope_ref(k_in, pos)
    ek, ev = hist_k.float().clone(), hist_v.float().clone()
    for b in range(B):
        ek[b, :, pos[b] % cap] = k_rot[b].float()
        ev[b, :, pos[b] % cap] = v_in[b].float()
    exact = F.scaled_dot_product_attention(q_rot.float()[:, :, None], ek, ev)[:, :, 0].reshape(B, Cd)
    amax_k, amax_v = hist_k.float().abs().amax(-1), hist_v.float().abs().amax(-1)
    k8, v8 = _encode(hist_k, amax_k, fmt).cuda(), _encode(hist_v, amax_v, fmt).cuda()
    ks, vs = (amax_k * (1.0 / qmax)).cuda(), (amax_v * (1.0 / qmax)).cuda()
    out = torch.empty(B, Cd, dtype=torch.bfloat16, device="cuda")
    qd, pd, md = qkv.cuda(), pos.cuda(), mask.cuda()
    _lib.check(lib.b200_op_attn_step_q8(cptr(qd), cptr(k8), cptr(v8), cptr(ks), cptr(vs), cptr(out), cptr(pd), cptr(md),
                                        B, H, cap, 0, 10000.0, kind, _stream()))
    kb, vb, out_b = hist_k.cuda(), hist_v.cuda(), torch.empty_like(out)
    _lib.check(lib.b200_op_attn_step(cptr(qd), cptr(kb), cptr(vb), cptr(out_b), cptr(pd), cptr(md), B, H, cap, 0, 10000.0, _stream()))
    torch.cuda.synchronize()
    rms = exact.pow(2).mean().sqrt()
    e_q8 = ((out.float().cpu() - exact).pow(2).mean().sqrt() / rms).item()
    e_bf = ((out_b.float().cpu() - exact).pow(2).mean().sqrt() / rms).item()
    print(f"{fmt} ring, key outlier channels x{outlier:g}: relative RMS error of the attention output {e_q8:.3%} (bf16 ring on the same data: {e_bf:.3%}); "
          f"ring bytes per session at context 3000, 32 layers: {32 * 2 * 3000 * 32 * (128 + 4) / 1e9:.3f} GB vs 1.573 GB")
    assert e_q8 < bound
