"""GPU: cross-attention conditioning of the temporal layers (LMModel(cross_attention=True), the TTS models' LM).

Kernels against fp64 (cross_attn_step_kernel, layernorm_kernel) and the condition memory's fill against the linear op it
runs; every layer's cross block against an fp64 restatement, teacher-forced on the taps, at batches that put the query and
output linears on each GEMM path; LMGen against the oracle (tests/cross_oracle.py, pinned on the reference by
tests/golden/lm_tiny_cross) with and without the graph, under CFG, with paused rows, across the ring wrap and through a
per-row condition swap and reset; the state, session records, paged and 8-bit rings; the int8 refusal."""
from __future__ import annotations

import ctypes as C
import json
from pathlib import Path

import pytest
import torch
from safetensors.torch import load_file

from tests.util import attn_ref64, cptr, greedy_unexcused, sampler_mismatches

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
COND = {"speaker_wavs": {"type": "tensor", "tensor": {"dim": 64}}}
FUSER = {"cross": ["speaker_wavs"], "cross_attention_pos_emb": True, "cross_attention_pos_emb_scale": 0.5}


def _lib():
    from moshi_b200 import _lib
    return _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _within(got: torch.Tensor, want: torch.Tensor) -> float:
    """worst |got - want| / (2^-7 |want| + 2^-8 rms), rms per row of the last dimension"""
    got, want = got.double().cpu(), want.double().cpu()
    rms = want.pow(2).mean(-1, keepdim=True).sqrt()
    return float(((got - want).abs() / (want.abs() * 2 ** -7 + rms * 2 ** -8 + 1e-30)).max())


# ---- kernels --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,H,T,nsplit", [(1, 2, 1, 1), (3, 16, 5, 0), (2, 32, 64, 3), (8, 16, 125, 0), (4, 2, 640, 0),
                                          (1, 16, 2000, 0), (256, 16, 125, 0), (5, 2, 2000, 1), (7, 32, 640, 16)])
def test_cross_attn_step_kernel_against_fp64(B, H, T, nsplit):
    lib = _lib().lib()
    g = torch.Generator().manual_seed(B * 1000 + T)
    q = torch.randn(B, H, 128, generator=g).bfloat16()
    k = torch.randn(B, H, T, 128, generator=g).bfloat16()
    v = torch.randn(B, H, T, 128, generator=g).bfloat16()
    ns = nsplit if nsplit > 0 else min(max(1, min(16, (148 * 4 + B * H - 1) // (B * H))), (T + 63) // 64)
    per = (T + ns - 1) // ns
    for b in range(B):                      # a needle key at the first, last and a split-edge position
        pos = [0, T - 1, min(per, T - 1)][b % 3]
        k[b, :, pos] = q[b]
    out = torch.empty(B, H * 128, dtype=torch.bfloat16, device="cuda")
    qd, kd, vd = q.cuda(), k.cuda(), v.cuda()
    _lib().check(lib.b200_op_cross_attn_step(cptr(qd), cptr(kd), cptr(vd), cptr(out), B, H, T, nsplit, _stream()))
    torch.cuda.synchronize()
    want = attn_ref64(q, k, v, [T] * B)
    ratio = _within(out.view(B, H, 128), want)
    print(f"cross attn B={B} H={H} T={T} nsplit={ns}: worst err / tolerance {ratio:.3f}")
    assert ratio <= 1.0


@pytest.mark.parametrize("M,dim", [(1, 256), (40, 2048), (130, 4096)])
def test_layernorm_kernel_against_fp64(M, dim):
    lib = _lib().lib()
    g = torch.Generator().manual_seed(dim + M)
    x = (torch.randn(M, dim, generator=g) * 3 + 0.5).bfloat16()
    w = (1 + 0.1 * torch.randn(dim, generator=g)).bfloat16()
    b = (0.05 * torch.randn(dim, generator=g)).bfloat16()
    y = torch.empty(M, dim, dtype=torch.bfloat16, device="cuda")
    xd_, wd, bd = x.cuda(), w.cuda(), b.cuda()
    _lib().check(lib.b200_op_layernorm(cptr(xd_), cptr(wd), cptr(bd), cptr(y), M, dim, _stream()))
    torch.cuda.synchronize()
    xd = x.double()
    want = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5) * w.double() + b.double()
    got = y.cpu().double()
    ulp = torch.pow(2.0, torch.floor(torch.log2(want.abs().clamp_min(1e-30))) - 7)
    assert bool(((got - want).abs() <= ulp).all())
    exact = float((got == want.bfloat16().double()).float().mean())
    print(f"layernorm M={M} dim={dim}: {exact:.5f} exactly rounded")
    assert exact >= 0.999


# ---- the handle ------------------------------------------------------------------------------------------------------------

def _cross_lm(fuser=FUSER, **over):
    from moshi_b200.config import tiny_lm_config
    from moshi_b200.models import LMModel
    from moshi_b200.synth import synth_lm_state_dict
    from oracle import scenarios
    cfg = tiny_lm_config(cross_attention=True, conditioners=COND, fuser=fuser, **over)
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    return cfg, sd, LMModel(cfg, sd, device="cuda")


def _voices(n: int, T: int, seed: int, short: int | None = None):
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    g = torch.Generator().manual_seed(seed)
    return [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(
        torch.randn(1, short if (short and b == 1) else T, 64, generator=g))}) for b in range(n)]


def _null(attrs):
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    out = []
    for a in attrs:
        t = a.tensor["speaker_wavs"].tensor
        out.append(ConditionAttributes(tensor={"speaker_wavs": TensorCondition(torch.zeros_like(t), torch.zeros(1, t.shape[1], dtype=torch.bool))}))
    return out


def _conditions(lm, attrs):
    ct = lm.condition_provider(lm.condition_provider.prepare(attrs))
    return ct, lm.fuser.get_cross(ct).to(torch.bfloat16).cpu()


@pytest.mark.parametrize("B", [40, 3])
def test_condition_fill_equals_the_linear_op(B):
    """k_cross / v_cross = the K|V rows of in_projs.0 through b200_op_linear_sk on the same 256-row chunks, reordered (B = 40:
    400 condition rows, a chunk edge inside row 25)."""
    lib = _lib().lib()
    cfg, sd, lm = _cross_lm()
    from moshi_b200.models import LMGen
    T, d = 10, cfg.dim
    ct, cross = _conditions(lm, _voices(B, T, seed=5))
    gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
    with gen.streaming(B):
        st = gen.get_streaming_state()
        src = cross.reshape(B * T, d).cuda().contiguous()
        for layer in range(cfg.num_layers):
            w = sd[f"transformer.layers.{layer}.cross_attention.in_projs.0.weight"][d:].cuda().contiguous()
            tiles = torch.empty(int(lib.b200_op_packed_bytes(2 * d, d, 0, 0)), dtype=torch.uint8, device="cuda")
            _lib().check(lib.b200_op_pack_tiles(cptr(w), cptr(tiles), 2 * d, d, 0, 0, _stream()))
            kv = torch.empty(B * T, 2 * d, dtype=torch.bfloat16, device="cuda")
            for i0 in range(0, B * T, 256):
                n = min(256, B * T - i0)
                chunk = src[i0:i0 + n].contiguous()
                out = torch.empty(n, 2 * d, dtype=torch.bfloat16, device="cuda")
                _lib().check(lib.b200_op_linear_sk(cptr(chunk), cptr(tiles), cptr(out), None, n, 2 * d, d, 0, 0, 0, 0, 0, _stream()))
                kv[i0:i0 + n] = out
            kv = kv.view(B, T, 2, cfg.num_heads, 128).permute(2, 0, 3, 1, 4).cpu()
            cx = st[f"lm_model.transformer.layers.{layer}.cross_attention"]
            assert torch.equal(cx.k_cross.cpu(), kv[0]) and torch.equal(cx.v_cross.cpu(), kv[1])
            want = (cross.double() @ w.cpu().double().t()).view(B, T, 2, cfg.num_heads, 128).permute(2, 0, 3, 1, 4)
            assert _within(cx.k_cross.cpu(), want[0]) <= 1.0


@pytest.mark.parametrize("B", [1, 3, 40, 130])
def test_cross_block_per_layer_against_fp64(B):
    """Each layer's x after the cross residual against fp64 LayerNorm, query, attention over the handle's own condition memory
    and out_proj, teacher-forced on the layer's x after the self-attention residual (tap)."""
    import torch.nn.functional as F
    cfg, sd, lm = _cross_lm()
    from moshi_b200.models import LMGen
    from oracle import scenarios
    ct, _ = _conditions(lm, _voices(B, 12, seed=B))
    gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
    codes = scenarios.lm_input_codes(cfg, B, 3, seed=B)
    d, H = cfg.dim, cfg.num_heads
    with gen.streaming(B):
        _lib().check(lm._lib.b200_lm_set_taps(lm._h, 1))
        worst = 0.0
        for i in range(3):
            gen.step(codes[i].cuda())
            st = gen.get_streaming_state()
            for l in range(cfg.num_layers):
                p = f"transformer.layers.{l}"
                x = gen.read_buffer(f"temporal.layers.{l}.x_attn", torch.bfloat16, (B, d)).cpu().double()
                got = gen.read_buffer(f"temporal.layers.{l}.x_cross", torch.bfloat16, (B, d)).cpu()
                cx = st[f"lm_model.transformer.{p.split('.', 1)[1]}.cross_attention"]
                xn = F.layer_norm(x, (d,), sd[p + ".norm_cross.weight"].double(), sd[p + ".norm_cross.bias"].double(), 1e-5)
                w = sd[p + ".cross_attention.in_projs.0.weight"].double()
                q = (xn @ w[:d].t()).view(B, H, 128)
                att = attn_ref64(q, cx.k_cross.cpu(), cx.v_cross.cpu(), [cx.k_cross.shape[2]] * B).reshape(B, d)
                upd = att @ sd[p + ".cross_attention.out_projs.0.weight"].double().t()
                want = x + upd
                err = (got.double() - want).abs() / (want.abs() * 2 ** -6 + upd.pow(2).mean(-1, keepdim=True).sqrt() * 2 ** -5)
                worst = max(worst, float(err.max()))
    print(f"cross block B={B}: worst err / tolerance {worst:.3f}")
    assert worst <= 1.0


def _gold():
    return load_file(GOLDEN / "lm_tiny_cross.safetensors"), json.loads((GOLDEN / "lm_tiny_cross.json").read_text())


def _run_pair(gen, orc, cfg, codes, info, g, name, *, tol, pause_row=None, check_sampling=False):
    """Steps the handle and the oracle side by side (oracle kept on the handle's tokens), with the fixture's per-row swap and
    reset; returns (worst text-logit diff, greedy flips unexcused, sampler mismatches)."""
    B = info["B"]
    worst, unexcused, smis = 0.0, 0, 0
    for i in range(info["steps"]):
        if i == info["reset_step"]:
            mask = torch.zeros(B, dtype=torch.bool)
            mask[info["swap_row"]] = True
            gen.set_condition_cross(g[name + ".swap_cross"], [info["swap_row"]])
            orc.set_condition_cross(g[name + ".swap_cross"], [info["swap_row"]])
            gen.reset_streaming(mask)
            orc.reset_streaming(mask)
        if pause_row is not None:
            m = torch.ones(B, dtype=torch.bool)
            m[pause_row] = not (3 <= i < 5)
            gen.set_exec_mask(m)
            orc.set_exec_mask(m)
        dbg: dict = {}
        noise = gen.draw_noise() if check_sampling else None
        kt, ka = min(gen.top_k_text, cfg.text_card), min(gen.top_k, cfg.card)
        orc.step(codes[i], None if noise is None else noise[:, :kt].cpu(),
                 None if noise is None else [noise[:, kt + k * ka:kt + (k + 1) * ka].cpu() for k in range(cfg.dep_q)], debug=dbg)
        gen.step(codes[i].cuda(), noise=noise)
        tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
        want = dbg["text_logits"].float()[:, 0, 0]
        worst = max(worst, (tl - want).abs().max().item())
        tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
        at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
        if check_sampling:
            smis += sampler_mismatches(tl, tt, True, gen.temp_text, gen.top_k_text, noise[:, :min(gen.top_k_text, cfg.text_card)].cpu())
        else:
            unexcused += greedy_unexcused(tt, dbg["text_token"], want, tol)[1]
        pos = orc.offsets % orc.cache.shape[2]
        for b in range(B):
            if orc.exec_mask[b]:
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    return worst, unexcused, smis


@pytest.mark.parametrize("fname,rname,use_graph,pause", [("cross", "greedy", True, False), ("cross_pos", "greedy", False, True),
                                                         ("cross_pos", "cfg", True, False), ("cross", "cfg", False, True),
                                                         ("cross_pos", "sampled", True, False)])
def test_lmgen_against_oracle(fname, rname, use_graph, pause):
    from moshi_b200.models import LMGen
    from oracle.lm import LMSpec
    from tests.cross_oracle import CrossLMOracle
    g, info = _gold()
    cfg, sd, lm = _cross_lm(fuser=info["fusers"][fname])
    run = info["runs"][rname]
    name = f"{fname}.{rname}"
    sampled = run["use_sampling"]
    B = info["B"]
    # the handle's own conditioners and fuser give the reference's condition (pinned on CPU); the fixture's is used below
    weights = {k[len(fname) + 1:]: v for k, v in g.items() if k.startswith(fname + ".condition_provider.")}
    from moshi_b200.conditioners import build_conditioning
    lm.condition_provider, lm.fuser = build_conditioning(cfg.conditioners, cfg.fuser, cfg.dim, weights, lm.device, True)
    from moshi_b200.conditioners import ConditionAttributes, TensorCondition
    attrs = [ConditionAttributes(tensor={"speaker_wavs": TensorCondition.from_tensor(g[f"voice.{b}"])}) for b in range(B)]
    if run["cfg_coef"] != 1.0:
        attrs += _null(attrs)
    ct = lm.condition_provider(lm.condition_provider.prepare(attrs))
    assert torch.equal(lm.fuser.get_cross(ct).to(torch.bfloat16).cpu(), g[name + ".condition_cross"])
    gen = LMGen(lm, use_sampling=sampled, cfg_coef=run["cfg_coef"], condition_tensors=ct)
    gen.use_graph = use_graph
    orc = CrossLMOracle(sd, LMSpec.from_config(cfg), condition_cross=g[name + ".condition_cross"].clone(), use_sampling=sampled,
                        cfg_coef=run["cfg_coef"], tie_break="index")
    orc.streaming(B)
    # 0.08 per model logit; the guided logits null + (l - null) * c combine two of them (lm.py:728-732)
    c = run["cfg_coef"]
    tol = 0.08 * (abs(c) + abs(1 - c)) if c != 1.0 else 0.08
    with gen.streaming(B):
        worst, unexcused, smis = _run_pair(gen, orc, cfg, g[f"{fname}.codes"], info, g, name, tol=tol, pause_row=2 if pause else None,
                                           check_sampling=sampled)
    print(f"{name} graph={use_graph} pause={pause}: worst text-logit diff {worst:.3e} (bound {tol:.2f}), unexcused flips {unexcused}, "
          f"sampler mismatches {smis}")
    assert worst <= tol and unexcused == 0 and smis == 0


def _steps(gen, codes, B, card, n):
    toks, logits = [], []
    for i in range(n):
        toks.append(gen.step(codes[i].cuda()))
        logits.append(gen.read_buffer("text_logits", torch.bfloat16, (B, card)).cpu())
    return torch.stack(logits), [t.cpu() if t is not None else None for t in toks]


def test_swap_changes_only_that_row_and_reset_keeps_memory():
    from moshi_b200.models import LMGen
    from oracle import scenarios
    cfg, sd, lm = _cross_lm()
    B, T = 3, 10
    ct, _ = _conditions(lm, _voices(B, T, seed=1))
    _, other = _conditions(lm, _voices(1, T, seed=2))
    codes = scenarios.lm_input_codes(cfg, B, 10, seed=3)
    runs = []
    for swap in (False, True):
        gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
        with gen.streaming(B):
            a, _ = _steps(gen, codes, B, cfg.text_card, 4)
            if swap:
                gen.set_condition_cross(other, [1])
            before = gen.get_streaming_state()["lm_model.transformer.layers.0.cross_attention"].k_cross.clone()
            gen.reset_streaming(torch.tensor([False, False, True]))
            after = gen.get_streaming_state()["lm_model.transformer.layers.0.cross_attention"].k_cross
            assert torch.equal(before, after)                    # _MHAState.reset keeps k_cross / v_cross
            b, _ = _steps(gen, codes[4:], B, cfg.text_card, 6)
        runs.append(torch.cat([a, b]))
    assert torch.equal(runs[0][:, [0, 2]], runs[1][:, [0, 2]])
    assert torch.equal(runs[0][:4], runs[1][:4]) and not torch.equal(runs[0][4:, 1], runs[1][4:, 1])


def test_state_round_trip_and_move_to_second_handle():
    from moshi_b200.models import LMGen
    from oracle import scenarios
    cfg, sd, lm = _cross_lm()
    from moshi_b200.models import LMModel
    lm2 = LMModel(cfg, sd, device="cuda")
    B = 3
    ct, _ = _conditions(lm, _voices(B, 10, seed=7))
    codes = scenarios.lm_input_codes(cfg, B, 14, seed=8)
    gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
    gen2 = LMGen(lm2, use_sampling=False, condition_tensors=_conditions(lm, _voices(B, 10, seed=70))[0])
    with gen.streaming(B), gen2.streaming(B):
        _steps(gen, codes, B, cfg.text_card, 6)
        snap = gen.get_streaming_state()
        assert "lm_model.transformer.layers.0.cross_attention" in snap
        want, _ = _steps(gen, codes[6:], B, cfg.text_card, 8)
        gen.set_streaming_state(snap)
        again, _ = _steps(gen, codes[6:], B, cfg.text_card, 8)
        gen2.set_streaming_state(snap)
        moved, _ = _steps(gen2, codes[6:], B, cfg.text_card, 8)
    assert torch.equal(want, again) and torch.equal(want, moved)


def test_session_records_carry_the_condition_memory():
    from moshi_b200.models import LMGen
    from oracle import scenarios
    cfg, sd, lm = _cross_lm()
    from moshi_b200.models import LMModel
    lm2 = LMModel(cfg, sd, device="cuda")
    B = 3
    ct, _ = _conditions(lm, _voices(B, 10, seed=11))
    codes = scenarios.lm_input_codes(cfg, B, 12, seed=12)
    gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
    gen2 = LMGen(lm2, use_sampling=False, condition_tensors=_conditions(lm, _voices(B, 10, seed=13))[0])
    with gen.streaming(B), gen2.streaming(B):
        _steps(gen, codes, B, cfg.text_card, 5)
        _steps(gen2, codes, B, cfg.text_card, 2)
        rec = gen.export_session(1)
        gen2.import_session(0, rec)
        codes2 = codes[5:].clone()
        codes2[:, 0] = codes[5:, 1]                              # row 0 of the second handle gets session 1's inputs
        want, _ = _steps(gen, codes[5:], B, cfg.text_card, 7)
        got, _ = _steps(gen2, codes2, B, cfg.text_card, 7)
    assert torch.equal(want[:, 1], got[:, 0])
    # refusals: another condition length, a handle without cross-attention
    gen3 = LMGen(lm2, use_sampling=False, condition_tensors=_conditions(lm, _voices(B, 9, seed=14))[0])
    with gen3.streaming(B):
        with pytest.raises(ValueError):
            gen3.import_session(0, rec)
    from moshi_b200.config import tiny_lm_config
    from moshi_b200.synth import synth_lm_state_dict
    plain_cfg = tiny_lm_config()
    plain = LMGen(LMModel(plain_cfg, synth_lm_state_dict(plain_cfg, seed=scenarios.LM_SEED), device="cuda"), use_sampling=False)
    with plain.streaming(B):
        with pytest.raises(ValueError):
            plain.import_session(0, rec)


def test_paged_ring_bit_identical_and_int8_ring_within_q8_tolerance():
    from moshi_b200.models import LMGen
    from oracle import scenarios
    from oracle.lm import LMSpec
    from tests.cross_oracle import CrossLMOracle
    cfg, sd, lm = _cross_lm()
    B = 3
    ct, cross = _conditions(lm, _voices(B, 10, seed=21))
    codes = scenarios.lm_input_codes(cfg, B, 16, seed=22)
    out = {}
    for kind in ("contiguous", "paged"):
        gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
        if kind == "paged":
            gen.kv_pool_frames, gen.kv_page_slots = B * cfg.context, 4
        with gen.streaming(B):
            out[kind] = _steps(gen, codes, B, cfg.text_card, 16)[0]
    assert torch.equal(out["contiguous"], out["paged"])
    gen = LMGen(lm, use_sampling=False, condition_tensors=ct)
    gen.kv_dtype = "int8"
    orc = CrossLMOracle(sd, LMSpec.from_config(cfg), condition_cross=cross, use_sampling=False, tie_break="index", kv_quant="int8")
    orc.streaming(B)
    worst, agree = 0.0, 0
    with gen.streaming(B):
        for i in range(16):
            dbg: dict = {}
            orc.step(codes[i], debug=dbg)
            gen.step(codes[i].cuda())
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            worst = max(worst, (tl - dbg["text_logits"].float()[:, 0, 0]).abs().max().item())
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            agree += int((tt == dbg["text_token"]).sum())
            pos = orc.offsets % orc.cache.shape[2]
            for b in range(B):
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print(f"int8 ring with cross-attention: worst text-logit diff {worst:.3e}, greedy text tokens equal {agree}/{16 * B}")
    assert worst < 0.12 and agree / (16 * B) > 0.9


def test_quantize_with_cross_attention_is_refused():
    from moshi_b200.config import LMConfig, tiny_lm_config
    with pytest.raises(ValueError):
        LMConfig.from_dict({**tiny_lm_config().to_reference_kwargs(), "cross_attention": True, "quantize": True,
                            "conditioners": COND, "fuser": FUSER})
    lib, L = _lib().lib(), _lib()
    from moshi_b200.models.lm import _config_struct
    c = _config_struct(tiny_lm_config(quantize=True))
    h = C.c_void_p()
    L.check(lib.b200_lm_create(C.byref(c), C.byref(h)))
    try:
        assert lib.b200_lm_set_cross_attention(h, 1) == L.B200_ERR_INVALID
    finally:
        lib.b200_lm_destroy(h)
