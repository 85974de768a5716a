"""Shared helpers for the GPU parity tests."""
from __future__ import annotations

import ctypes as C
import functools
import math

import numpy as np
import torch
import torch.nn.functional as F


def stats(name: str, got: torch.Tensor, want: torch.Tensor) -> str:
    got, want = got.detach().float().cpu(), want.detach().float().cpu()
    diff = (got - want).abs()
    scale = want.abs().max().item() + 1e-30
    return (f"{name}: max_abs={diff.max().item():.3e} rel_to_max={diff.max().item() / scale:.3e} "
            f"ref_std={want.std().item():.3e} nan={int(torch.isnan(got).sum())}")


def rvq_mismatches(codes_got: torch.Tensor, codes_want: torch.Tensor, margins: torch.Tensor,
                   n_semantic: int = 1, tol: float = 1e-4):
    """Margin-aware comparison of RVQ indices ([B, K, T] each).

    A mismatch at level k is excused iff the oracle's own relative gap between the best and the
    second-best squared distance at that level is below ``tol`` (a rounding-order tie) or an earlier
    level of the same quantizer already flipped (the residual, hence every later index, differs).
    Returns (n_mismatch, n_unexcused).
    """
    got, want = codes_got.cpu(), codes_want.cpu()
    B, K, T = want.shape
    bad = unexcused = 0
    for b in range(B):
        for t in range(T):
            for lo, hi in ((0, n_semantic), (n_semantic, K)):
                flipped = False
                for k in range(lo, hi):
                    if got[b, k, t] != want[b, k, t]:
                        bad += 1
                        if not flipped and margins[b, k, t] > tol:
                            unexcused += 1
                        flipped = True
    return bad, unexcused


def cptr(t: torch.Tensor | None) -> C.c_void_p:
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def greedy_unexcused(got: torch.Tensor, want: torch.Tensor, logits_oracle: torch.Tensor, tol: float) -> tuple[int, int]:
    """Margin-aware comparison of greedy ids ([N] each) against the oracle's fp32-viewed logits ([N, card]): a mismatch is
    excused iff the oracle's own top-2 logit gap is below ``2 * tol`` (two logits that each moved by <= tol can swap).
    Returns (n_mismatch, n_unexcused)."""
    top2 = logits_oracle.float().topk(2, dim=-1).values
    gap = top2[:, 0] - top2[:, 1]
    bad = got.cpu() != want.cpu()
    return int(bad.sum()), int((bad & (gap > 2 * tol)).sum())


def sampler_mismatches(logits: torch.Tensor, toks: torch.Tensor, sampling: bool, temp: float, top_k: int,
                        noise: torch.Tensor | None) -> int:
    """Tokens that differ from the reference sampler run on the device's own logits [B, card] with the same noise.  A
    difference is excused only where the two best candidates' scores p / q agree to fp32 rounding (relative 1e-5)."""
    from oracle.lm import sample_token
    want = sample_token(logits.float(), sampling, temp, top_k, noise, tie_break="index")
    bad = (want != toks).nonzero().flatten().tolist()
    n = 0
    for b in bad:
        if sampling:
            lg = logits[b].double()
            srt = torch.sort(lg, descending=True, stable=True)
            k = min(top_k, lg.numel())
            score = torch.softmax(srt.values / temp, -1)[:k] / noise[b, :k].double()
            top2 = score.topk(2).values
            if float((top2[0] - top2[1]) / top2[0]) < 1e-5:
                continue
        n += 1
    return n


def sample_is_stable(logits: torch.Tensor, temp: float, top_k: int, noise: torch.Tensor, tol: float) -> torch.Tensor:
    """For every row of oracle logits ([N, card], fp32 view of the bf16 tensor) with its Exp(1) noise ([N, k]): is the
    sampled token (sampling.py:86-106: softmax(l / temp) -> top-k -> argmax(p / q), noise indexed by RANK) the same for
    every logit vector within ``tol`` (max-norm) of this one?  Conservative test:
      * a candidate's log-probability moves by at most 2 * tol / temp (its logit and the normaliser);
      * candidates whose logits lie in one run of the sorted order with adjacent gaps < 2 * tol can exchange ranks, i.e. any
        of them can receive any noise value of that run (this also covers exact ties, whose torch.topk order is unspecified,
        and candidates that can cross the top-k boundary).
    Stable iff the winner's worst-case score exceeds every other candidate's best-case score.  Returns bool [N]."""
    logits = logits.float().cpu()
    noise = noise.float().cpu()
    N, card = logits.shape
    k = min(top_k, card)
    out = torch.zeros(N, dtype=torch.bool)
    for n in range(N):
        srt, _ = torch.sort(logits[n], descending=True, stable=True)
        logp = torch.log_softmax(srt / temp, dim=-1)
        q = torch.cat([noise[n, :k], torch.full((card - k,), float("inf"))])     # ranks beyond k never win
        score = logp[:k] - torch.log(noise[n, :k])
        w = int(score.argmax())
        # runs of the sorted order whose adjacent gaps are all < 2 * tol
        brk = torch.cat([torch.tensor([True]), (srt[:-1] - srt[1:]) >= 2 * tol])
        run_id = torch.cumsum(brk.int(), 0) - 1
        n_runs = int(run_id[-1]) + 1
        qmin = torch.full((n_runs,), float("inf")).scatter_reduce(0, run_id, q, reduce="amin")
        qmax = torch.full((n_runs,), 0.0).scatter_reduce(0, run_id, q, reduce="amax")
        slack = 2 * tol / temp
        best_case = logp + slack - torch.log(qmin[run_id])          # every candidate, with the smallest noise it could be dealt
        worst_w = logp[w] - slack - torch.log(qmax[run_id[w]])      # the winner, with the largest noise it could be dealt
        best_case[w] = -float("inf")
        if int((run_id == run_id[w]).sum()) > 1:                    # the winner itself can be re-ranked: not stable
            continue
        out[n] = bool(worst_w > best_case.max())
    return out


def to_candle_layout(cfg, sd: dict) -> dict:
    """The Rust / candle checkpoint layout of the LM (``scripts/import_rust.py:45-113``, what ``rust/moshi-core`` loads): the
    temporal transformer under the reference's names, the depformer per codebook step as ``depformer.<k>.*``."""
    out = {k: v for k, v in sd.items() if k.startswith(("text_emb", "text_linear", "out_norm", "emb.", "transformer.", "extra_heads."))}
    for k in range(cfg.dep_q):
        base = f"depformer.{k}."
        out[base + "linear_in.weight"] = sd[f"depformer_in.{k}.weight"]
        out[base + "linear_out.weight"] = sd[f"linears.{k}.weight"]
        out[base + "emb.weight"] = sd["depformer_text_emb.weight"] if k == 0 else sd[f"depformer_emb.{k - 1}.weight"]
        for layer in range(cfg.depformer_num_layers):
            src, dst = f"depformer.layers.{layer}.", base + f"transformer.layers.{layer}."
            out[dst + "self_attn.in_proj_weight"] = sd[src + f"self_attn.in_projs.{k}.weight"]
            out[dst + "self_attn.out_proj.weight"] = sd[src + f"self_attn.out_projs.{k}.weight"]
            out[dst + "norm1.alpha"] = sd[src + "norm1.alpha"]
            out[dst + "norm2.alpha"] = sd[src + "norm2.alpha"]
            out[dst + "gating.linear_in.weight"] = sd[src + f"gating.{k}.linear_in.weight"]
            out[dst + "gating.linear_out.weight"] = sd[src + f"gating.{k}.linear_out.weight"]
    return out


# ---- fp64 references of the LM's attention and RMSNorm kernels -------------------------------------------------------------
def rope_ref(x: torch.Tensor, pos: torch.Tensor, max_period: float = 10000.0) -> torch.Tensor:
    """rope.py:45-82 on [B, H, D] bf16 for one time step at per-row position ``pos``: interleaved pairs, fp32, -> bf16.

    The angle is fp32(freq) * fp32(pos) as in the reference, so a position past 2^24 rounds the way the reference's does (a
    float64 angle would not).  freq, cos and sin are the correctly rounded fp32 values of the fp32 arguments (taken in
    float64): torch's vectorised CPU exp is one ulp off for one of the 64 frequencies, and at position 2^24 one ulp of a
    frequency turns the angle by a radian."""
    B, H, D = x.shape
    xf = x.float().view(B, H, D // 2, 2)
    arg = torch.arange(D // 2, dtype=torch.float32) * torch.tensor(-math.log(max_period) * 2 / D, dtype=torch.float32)
    freqs = torch.exp(arg.double()).float()
    theta = (freqs[None, :] * pos.float()[:, None]).double()
    c, s_ = torch.cos(theta).float()[:, None, :], torch.sin(theta).float()[:, None, :]
    xr, xi = xf[..., 0], xf[..., 1]
    return torch.stack([xr * c - xi * s_, xr * s_ + xi * c], dim=-1).view(B, H, D).bfloat16()


def attn_ref64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, n_valid, scale: float | None = None) -> torch.Tensor:
    """softmax(scale * q . k) . v over the slots [0, n_valid[b]) of each row, in float64: q [B, H, D], k / v [B, H, S, D]
    -> [B, H, D].  The valid slots are selected explicitly (no masked SDPA: a NaN in a masked slot would leak through
    0 * NaN), and a row without a valid key gives zeros, which is what the kernels write."""
    B, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    out = torch.zeros(B, H, D, dtype=torch.float64)
    for b in range(B):
        n = int(n_valid[b])
        if n == 0:
            continue
        kk, vv = k[b, :, :n].double(), v[b, :, :n].double()
        s = torch.einsum("hd,hnd->hn", q[b].double(), kk) * scale
        out[b] = torch.einsum("hn,hnd->hd", torch.softmax(s, dim=-1), vv)
    return out


def rmsnorm_ref64(x: torch.Tensor, alpha: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """transformer.py:45-58 in float64: x * alpha / sqrt(eps + mean(x^2)) over the last dimension."""
    x = x.double()
    return x * alpha.double() / torch.sqrt(eps + x.pow(2).mean(-1, keepdim=True))


# Acceptance rule of the attention outputs: |got - want| <= ATTN_REL * |want| + c * rms(want over the head's D outputs).
# ATTN_REL is twice the largest bf16 rounding of the output (half an ulp is 2^-8 of the value at the bottom of a binade); c is
# what fp32 arithmetic adds on top (the bf16 kernels: ATTN_C).  A single lost key out of 3000 moves the largest output of a head
# by about 0.05 rms, so every c used here stays far below that.
ATTN_REL = 2.0 ** -7
ATTN_C = 2.0 ** -8


def err_ratios(got: torch.Tensor, want: torch.Tensor, c: float = ATTN_C) -> torch.Tensor:
    """|got - want| / (ATTN_REL |want| + c rms(want over the last dimension)) per element (<= 1 passes).  Where the tolerance
    is 0 (a row with no valid key) only an exact zero passes; a NaN never does."""
    want = want.detach().double()
    got = got.detach().to(want.device, torch.float64).reshape(want.shape)
    err = (got - want).abs()
    tol = ATTN_REL * want.abs() + c * want.pow(2).mean(-1, keepdim=True).sqrt()
    ratio = torch.where(tol > 0, err / tol, torch.where(err <= 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    return torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)


def attn_err_ratio(got: torch.Tensor, want: torch.Tensor, c: float = ATTN_C) -> float:
    """Largest err_ratios over all outputs (<= 1 passes)."""
    return float(err_ratios(got, want.cpu(), c).max())


def close_to_ref(got: torch.Tensor, want: torch.Tensor, c: float = ATTN_C) -> bool:
    return attn_err_ratio(got, want, c) <= 1.0


# ---- scenarios of one temporal attention step ----------------------------------------------------------------------------
BF16_NAN = 0x7FC0            # a quiet bf16 NaN, as int16


def attn_pick_splits(B: int, H: int, cap: int) -> int:
    """The LM's split count for a (B, H, cap) step (lm_kernels.cuh attn_pick_splits)."""
    ns = min(max(-(-592 // (B * H)), 1), 16)
    return min(ns, -(-cap // 64))


def split_ranges(n_valid: int, nsplit: int) -> list[tuple[int, int]]:
    """The key ranges [s0, s1) of the kernel's splits for a row with n_valid keys (empty ranges included)."""
    per = -(-n_valid // nsplit)
    return [(min(j * per, n_valid), min((j + 1) * per, n_valid)) for j in range(nsplit)]


def attn_rows(cap: int, nsplit: int) -> list[tuple[int, int]]:
    """(pos, exec) of the rows of a scenario: fills at the 32-key group and 64-key loop-step edges, fewer keys than splits,
    around a middle split boundary, cap - 1 and cap; new keys landing on the first slot, the last slot of split 0 and the first
    slot of split 1 of a wrapped ring, one hour at 12.5 Hz; paused rows young, full, wrapped and empty.

    No position reaches 2^24: there one ulp of a RoPE frequency turns the angle by a radian, and the kernel's fp32 exp / sincos
    and any host fp32 reference disagree on a few of the 64 frequencies, so no reference can pin the kernel down."""
    per = -(-cap // nsplit)
    j = max(nsplit // 2, 1)
    fills = [1, 31, 32, 33, 63, 64, 65, nsplit - 1, per * j - 1, per * j, per * j + 1, cap - 1, cap]
    rows = [(n - 1, 1) for n in fills if 1 <= n <= cap]
    rows += [(p, 1) for p in (cap, cap + per - 1, cap + per, 45000)]
    rows += [(max(cap // 3, 1), 0), (cap, 0), (2 * cap + 7, 0), (0, 0)]
    return list(dict.fromkeys(rows))


@functools.lru_cache(maxsize=4)
def _ring_base(H: int, cap: int, D: int, seed: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Four rings of N(0, 1) keys and values that the rows of a scenario share (saves the host time of generating each)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(4, H, cap, D, generator=g).bfloat16(), torch.randn(4, H, cap, D, generator=g).bfloat16())


def attn_scenario(H: int, cap: int, nsplit: int, *, D: int = 128, seed: int = 0, qk_scale: float = 1.0, v_scale: float = 1.0,
                  q_scale: float = 1.0, needles: bool = True, extra_needles: tuple[int, ...] = (), needle_score: float = 12.0) -> dict:
    """Inputs of one attention step over the rows of ``attn_rows`` and what the step must produce.

    * Rings hold N(0, 1) keys (already rotated) and values on the slots written so far.  Young rings hold bf16 NaN at and after
      the slot the step writes, and a paused row's unwritten slot is NaN too: the kernel must neither read nor change them.
    * Needles: keys lined up with the row's rotated query (score ``needle_score``, about +10 over the rest) with values of
      4 N(0, 1), on the first and last slot of every split, on slot n_valid - 1, on the oldest key of a full ring and on
      ``extra_needles``.  The new key is a
      needle (k_in = alpha * q_in).  In a wrapped ring the OLD key at pos % cap is a needle too: an executing row must not
      attend to it (the step overwrites it), a paused row must.
    Returns qkv [B, 3 H D] bf16, rings k / v [B, H, cap, D] bf16 (before the step), pos, mask, nsplit (resolved), n_valid,
    q_rot / k_rot (fp32-RoPE reference), k_ref / v_ref (the rings after the step) and want = attn_ref64 [B, H, D]."""
    rows = attn_rows(cap, nsplit if nsplit > 0 else attn_pick_splits(24, H, cap))
    B = len(rows)
    ns = nsplit if nsplit > 0 else attn_pick_splits(B, H, cap)
    pos = torch.tensor([p for p, _ in rows], dtype=torch.int64)
    mask = torch.tensor([e for _, e in rows], dtype=torch.bool)
    n_valid = (pos + mask.long()).clamp(max=cap)
    g = torch.Generator().manual_seed(seed * 7919 + H * 131 + cap * 17 + ns)
    C = H * D
    qkv = torch.randn(B, 3 * C, generator=g)
    qkv[:, :2 * C] *= qk_scale
    qkv[:, :C] = (qkv[:, :C] * q_scale).clamp(-256, 256)       # q_scale: queries alone, at most 256 per element
    qkv[:, 2 * C:] *= v_scale
    qkv = qkv.bfloat16()
    q_in, k_in, v_in = (qkv[:, i * C:(i + 1) * C].reshape(B, H, D) for i in range(3))
    q_rot = rope_ref(q_in, pos)
    base_k, base_v = _ring_base(H, cap, D, seed)
    k = torch.empty(B, H, cap, D, dtype=torch.bfloat16)
    v = torch.empty_like(k)
    for b in range(B):
        written = min(int(pos[b]), cap)                          # slots holding a key before the step
        k[b].view(torch.int16).fill_(BF16_NAN)
        v[b].view(torch.int16).fill_(BF16_NAN)
        k[b, :, :written] = (base_k[b % 4, :, :written].float() * qk_scale).bfloat16()
        v[b, :, :written] = (base_v[b % 4, :, :written].float() * v_scale).bfloat16()
    if needles:
        qn = q_rot.float()
        # a key lined up with q whose score is needle_score: k = q * needle_score * sqrt(D) / |q|^2
        k_needle = (qn * (needle_score * D ** 0.5 / qn.pow(2).sum(-1, keepdim=True))).bfloat16()     # [B, H, D]
        for b in range(B):
            p, n, ex = int(pos[b]), int(n_valid[b]), bool(mask[b])
            if n == 0:
                continue
            slots = {s for s0, s1 in split_ranges(n, ns) if s1 > s0 for s in (s0, s1 - 1)} | {n - 1}
            slots |= {s for s in extra_needles if s < n}
            if p >= cap:
                slots.add(p % cap)                               # the old key: overwritten by an executing row
            if n == cap:
                slots.add((p + ex) % cap)                        # the oldest key the step attends to
            if ex and p < cap:
                slots.discard(p)                                 # a young ring's new slot is poison until the step writes it
            for s in sorted(slots):
                k[b, :, s] = k_needle[b]
                v[b, :, s] = (torch.randn(H, D, generator=g) * 4 * v_scale).bfloat16()
        # the new key: k_in = alpha * q_in, with alpha chosen so that its rotated score is needle_score
        qf = q_in.float()
        alpha = needle_score * D ** 0.5 / qf.pow(2).sum(-1, keepdim=True)
        k_in_new = (qf * alpha).bfloat16()
        v_in_new = (torch.randn(B, H, D, generator=g) * 4 * v_scale).bfloat16()
        qkv = qkv.view(B, 3, H, D).clone()
        qkv[:, 1], qkv[:, 2] = k_in_new, v_in_new
        qkv = qkv.view(B, 3 * C)
        k_in, v_in = k_in_new, v_in_new
    k_rot = rope_ref(k_in, pos)
    k_ref, v_ref = k.clone(), v.clone()
    for b in range(B):
        if mask[b]:
            k_ref[b, :, int(pos[b]) % cap] = k_rot[b]
            v_ref[b, :, int(pos[b]) % cap] = v_in[b]
    want = attn_ref64(q_rot, k_ref, v_ref, n_valid)
    return dict(H=H, cap=cap, D=D, B=B, nsplit=ns, qkv=qkv, k=k, v=v, pos=pos, mask=mask, n_valid=n_valid, q_rot=q_rot,
                k_rot=k_rot, k_ref=k_ref, v_ref=v_ref, want=want)


# The 8-bit ring kernel forms q.k and the weighted value sums in fp16 (HFMA2, four products per lane partial): its outputs get
# this much more room per rms on top of ATTN_C.
Q8_FP16_C = 2.0 ** -8
# At the end of its supported query range (|q| = 256 per element) the scores are in the hundreds: their fp16 rounding (~2^-11
# of sum |q_i k_i|) and a RoPE angle that differs in its last fp32 bits move them by tenths, so near-tied keys trade weight.
# There the outputs are only checked to stay finite and within this much per rms (measured worst: 2.2 x 2^-4 on e4m3).
Q8_WIDE_C = 2.0 ** -2


def dep_scenario(B: int, H: int, dep_q: int, seed: int = 0, needle_score: float = 12.0) -> dict:
    """Inputs of the depformer attention sub-steps 0..dep_q - 1 on one per-frame cache (D = 64, scale 1/8, no RoPE).  Every
    query has two needles: key 0 (each query carries a component along k_0) and its own new key (k_s = alpha q_s).  Returns
    qkv [dep_q, B, 3 H 64] bf16 and want [dep_q, B, H, 64] = attn_ref64 over keys 0..s."""
    D = 64
    g = torch.Generator().manual_seed(seed * 31 + B * 7 + H + dep_q)
    q = torch.randn(dep_q, B, H, D, generator=g)
    v = torch.randn(dep_q, B, H, D, generator=g).bfloat16()
    k0 = torch.randn(B, H, D, generator=g)
    q[1:] += k0 * (needle_score * 8 / k0.pow(2).sum(-1, keepdim=True))
    q = q.bfloat16()
    qf = q.float()
    k = (qf * (needle_score * 8 / qf.pow(2).sum(-1, keepdim=True))).bfloat16()
    k[0] = k0.bfloat16()
    qkv = torch.cat([q, k, v], dim=2).reshape(dep_q, B, 3 * H * D)     # rows q (h d) | k (h d) | v (h d)
    ks, vs = k.permute(1, 2, 0, 3), v.permute(1, 2, 0, 3)            # [B, H, dep_q, D]
    want = torch.stack([attn_ref64(q[s], ks, vs, [s + 1] * B, scale=0.125) for s in range(dep_q)])
    return dict(B=B, H=H, D=D, dep_q=dep_q, qkv=qkv, q=q, k=ks, v=vs, want=want)


def rmsnorm_verdict(got: torch.Tensor, x: torch.Tensor, alpha: torch.Tensor) -> tuple[float, float]:
    """(largest distance of ``got`` from bf16(rmsnorm_ref64(x, alpha)) in bf16 ulps of the latter, share of equal elements)."""
    want = rmsnorm_ref64(x, alpha).bfloat16().float()
    g = got.detach().cpu().bfloat16().float()
    ulp = torch.where(want != 0, 2.0 ** (torch.floor(torch.log2(want.abs())) - 7), torch.full_like(want, 2.0 ** -133))
    d = torch.nan_to_num((g - want).abs() / ulp, nan=math.inf, posinf=math.inf)
    return float(d.max()), float((g == want).float().mean())


# ---- fp64 reference of one depformer frame ---------------------------------------------------------------------------------
def _bf(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 and back (a cast point of the bf16 model), to nearest with ties to even.  torch casts float64 to bf16
    through float32, which turns a value within half a float32 ulp of a bf16 midpoint into a tie and can round it the wrong
    way; float64 input therefore goes to float32 rounded to odd (toward zero, then the last bit set where inexact), after
    which float32 -> bf16 rounds correctly."""
    if x.dtype != torch.float64:
        return x.to(torch.bfloat16).to(x.dtype)
    f = x.float()
    f = torch.where(f.double().abs() > x.abs(), torch.nextafter(f, torch.zeros_like(f)), f)
    f = torch.where(f.double() != x, (f.view(torch.int32) | 1).view(torch.float32), f)
    return f.to(torch.bfloat16).to(x.dtype)


def _dep_tensor(sd: dict, name: str, k: int, layer: int | None) -> torch.Tensor:
    """The state-dict tensor of the depformer's weight ``name`` at sub-step k (and layer)."""
    p = f"depformer.layers.{layer}."
    key = {"din": f"depformer_in.{k}.weight",
           "emb": "depformer_text_emb.weight" if k == 0 else f"depformer_emb.{k - 1}.weight",
           "in": p + f"self_attn.in_projs.{k}.weight", "out": p + f"self_attn.out_projs.{k}.weight",
           "lin_in": p + f"gating.{k}.linear_in.weight", "lin_out": p + f"gating.{k}.linear_out.weight",
           "n1": p + "norm1.alpha", "n2": p + "norm2.alpha", "head": f"linears.{k}.weight"}[name]
    return sd[key]


@torch.no_grad()
def depformer_ref64(sd: dict, cfg, transformer_out: torch.Tensor, text_token: torch.Tensor, audio_tokens: torch.Tensor,
                    mutant: dict | None = None, quantize: bool = False, din: torch.Tensor | None = None) -> dict:
    """One depformer frame (lm.py:450-493 and 809-850 with transformer.py's weights-per-step layers, as oracle/lm.py
    forward_depformer / depformer_step state it) in float64, teacher-forced: sub-step k's previous token is ``text_token`` [B]
    for k = 0 and ``audio_tokens[k - 1]`` ([dep_q, B], the tokens the model under test sampled) after.  Values are rounded to
    bf16 at the cast points of the bf16 model (csrc/dep_fused.cu):
      x = bf16(bf16(din_k) + emb_k(prev));  xn = bf16(rmsnorm(x));  q, k, v = bf16(in_proj(xn));
      out = bf16(softmax(q . k_j / 8) . v_j over the keys j = 0..k);  x = bf16(x + bf16(out_proj(out)));
      h = bf16(bf16(silu(bf16 g)) * bf16 u);  x = bf16(x + bf16(linear_out(h)));  logits = linears[k](x).
    Runs on transformer_out's device.  Weights are converted to float64 one (sub-step, layer) at a time, never all at once.

    ``quantize`` (LMModel(quantize=True), every linear a QLinear): each linear of the frame (din, in, out, lin_in, lin_out and
    head) is oracle/quant.py's restatement on the bf16 value at its cast point: the activation rows quantised in fp32 with
    ties to even, the weight rows quantised through fp16 once (quant.cached_quantize_weight; the gate and value rows of lin_in
    keep their own scales), the exact integer product, dequantised in qlinear_f32's fp32 order.  The RMSNorm, the attention
    and the SiLU stay float64.

    ``din`` (bf16 [B, dep_q, dd], the device's own din) teacher-forces every sub-step's input on it: the returned "din" is still
    depformer_in[k] of transformer_out, to judge the device's din by.

    Returns the checkpoints before their final bf16 rounding, as float64: "din" [B, dep_q, dd] (depformer_in[k] of
    transformer_out), "k" / "v" per layer [B, H, dep_q, 64] (what the layer's per-frame cache holds after the frame) and
    "logits" [dep_q, B, card].

    ``mutant`` (for the tests of the acceptance rule) replaces parts of the computation:
      "weight": f(name, k, layer, fetch) -> the raw tensor to use, where fetch(name, k, layer) gives the right one (names:
                din, emb, in, out, lin_in, lin_out, n1, n2, head);
      "keys":   f(k, layer) -> (lo, hi): the keys the sub-step attends over (default (0, k + 1));
      "prev":   f(k, tokens) -> the previous tokens of sub-step k, tokens = [text_token, audio_tokens[0], ...];
      "residual": f(k, layer, "attn" | "ffn") -> False to drop that residual;
      "qlinear": f(name, k, layer, x, q) -> q (quantize only): q = dict(qx, sa, qw, sw) holds the quantised activation rows,
                 their scales, the quantised weight and its row scales of that linear, x its bf16 input."""
    mutant = mutant or {}
    dev, f64 = transformer_out.device, torch.float64
    B = transformer_out.shape[0]
    dd, H, L, Q = cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_num_layers, cfg.dep_q
    D = dd // H

    def fetch(name, k, layer=None):
        return _dep_tensor(sd, name, k, layer)

    def raw(name, k, layer=None):
        return mutant["weight"](name, k, layer, fetch) if "weight" in mutant else fetch(name, k, layer)

    def W(name, k, layer=None):
        t = raw(name, k, layer)
        if name == "emb":
            return t                                    # only the rows of the previous tokens are gathered and converted
        t = t.to(dev, f64)
        return t.reshape(-1) if name in ("n1", "n2") else t

    def lin(x, name, k, layer=None):
        """x . w^T of one linear for bf16-valued x, before the output's rounding."""
        if not quantize:
            return x @ W(name, k, layer).T
        from oracle.quant import cached_quantize_weight, qproduct_f32, quantize_rows
        xb = x.to(torch.bfloat16)
        qx, sa = quantize_rows(xb)
        qw, sw = cached_quantize_weight(raw(name, k, layer).to(dev))
        q = dict(qx=qx, sa=sa, qw=qw, sw=sw)
        if "qlinear" in mutant:
            q = mutant["qlinear"](name, k, layer, xb, q)
        return qproduct_f32(q["qx"], q["sa"], q["qw"], q["sw"]).to(f64)

    def rmsnorm(x, alpha):
        return _bf(x * alpha / torch.sqrt(1e-8 + x.pow(2).mean(-1, keepdim=True)))

    tout = transformer_out.to(f64)
    tokens = [text_token.to(dev)] + [audio_tokens[k].to(dev) for k in range(Q - 1)]
    din_in = din
    din = torch.stack([lin(tout, "din", k) for k in range(Q)], dim=1)
    x_din = din if din_in is None else din_in.to(dev, f64)
    kc = [torch.zeros(B, H, Q, D, dtype=f64, device=dev) for _ in range(L)]
    vc = [torch.zeros(B, H, Q, D, dtype=f64, device=dev) for _ in range(L)]
    logits = []
    for k in range(Q):
        prev = mutant["prev"](k, tokens) if "prev" in mutant else tokens[k]
        table = W("emb", k)
        e = table.to(dev)[prev.clamp(min=0)].to(f64) * (prev >= 0)[:, None]          # token -1 -> zero row (lm_utils.py:103-121)
        x = _bf(_bf(x_din[:, k]) + e)
        for layer in range(L):
            xn = rmsnorm(x, W("n1", k, layer))
            qkv = lin(xn, "in", k, layer).view(B, 3, H, D)
            kc[layer][:, :, k], vc[layer][:, :, k] = qkv[:, 1], qkv[:, 2]
            lo, hi = mutant["keys"](k, layer) if "keys" in mutant else (0, k + 1)
            s = torch.einsum("bhd,bhnd->bhn", _bf(qkv[:, 0]), _bf(kc[layer][:, :, lo:hi])) * 0.125
            o = _bf(torch.einsum("bhn,bhnd->bhd", torch.softmax(s, dim=-1), _bf(vc[layer][:, :, lo:hi]))).reshape(B, dd)
            upd = _bf(lin(o, "out", k, layer))
            x = _bf(x + upd) if mutant.get("residual", lambda *a: True)(k, layer, "attn") else upd
            xn = rmsnorm(x, W("n2", k, layer))
            gu = lin(xn, "lin_in", k, layer)
            F_ = gu.shape[1] // 2
            g, u = _bf(gu[:, :F_]), _bf(gu[:, F_:])
            h = _bf(_bf(g * torch.sigmoid(g)) * u)
            upd = _bf(lin(h, "lin_out", k, layer))
            x = _bf(x + upd) if mutant.get("residual", lambda *a: True)(k, layer, "ffn") else upd
        logits.append(lin(x, "head", k))                                             # depformer_norms is Identity (lm.py:197-198)
    return dict(din=din, k=kc, v=vc, logits=torch.stack(logits))


# Acceptance rule of the depformer checkpoints: err_ratios with the rms taken per (row, head) for k / v and per row for din and
# logits, and one c per checkpoint kind.  Each c is about twice what the bf16 oracle (oracle/lm.py: an independent bf16
# implementation, fp32 accumulation in another order) needs against depformer_ref64 at the 7B depformer shapes (dd 1024,
# 16 heads, ffn 2816, 6 layers, dep_q 8, card 2048), B = 4, two frames of a random N(0, 1) transformer_out, teacher-forced on
# the oracle's own greedy tokens (tests/test_depformer_ref_cpu.py measures it again and asserts that the oracle passes).
# Rounding flips random-walk through the layers, so the k / v constant grows with depth: DEP_C_KV[l] for layer l (the last
# entry for deeper layers).  What the oracle needs (c_needed):
#   din 0 (every output within the relative term), k / v of layers 0..5: 0.0004, 0.0125, 0.0196, 0.0244, 0.0309, 0.0466,
#   logits 0.0402.
# Layer 0's k / v carry no random walk yet, only the rare bf16 flips of din and of the RMSNorm output, so four rows sample their
# tail poorly: at B = 256 (two frames, the same test file) the oracle needs 0.0015 there (0.0019 with other draws), and
# layer 0 gets 2^-8, twice the larger.  din gets
# a floor of 2^-10 of the rms for fp32 accumulation in another order.
# The 2B depformer (the same layer shapes, dep_q 16 sub-steps, depformer_in with K 2560) needs din 0, k / v 0.0002, 0.0126,
# 0.0252, 0.0261, 0.0394, 0.0401, logits 0.0387, and 0.0019 at layer 0 at B = 256: layers 2 and 4 (0.04 and 0.0625 from the
# 7B shapes, 1.6 times what they need there) get 0.05 and 0.08.  (Measured with _bf rounding float64 correctly; the 7B
# numbers above were taken with torch's cast, which rounds through float32, and move by at most 0.005 with it.)
DEP_C_DIN = 2.0 ** -10
DEP_C_KV = (2.0 ** -8, 0.025, 0.05, 0.05, 0.08, 0.094)
DEP_C_LOGITS = 0.08
# int8 (quantize=True, depformer_ref64(quantize=True)): din is exact given transformer_out and is checked bit for bit.  An
# activation one bf16 ulp away from the reference's that sits on a rounding boundary of the row quantiser moves by a whole int8
# step (about absmax / 127, several bf16 ulps of the rms), so the random walk through the layers is wider than in bf16.  The
# int8 oracle on dep_row_scaled weights (the same shapes, B = 4, two frames, three draws) needs: k / v of layers 0..5 0,
# 0.126, 0.237, 0.240, 0.251, 0.313, logits 0.257; layer 0 at B = 256 needs 0.0033.  Each constant is about twice that.
DEP_C_KV_I8 = (2.0 ** -7, 0.25, 0.5, 0.5, 0.5, 0.625)
DEP_C_LOGITS_I8 = 0.5


def dep_c_kv(layer: int, int8: bool = False) -> float:
    c = DEP_C_KV_I8 if int8 else DEP_C_KV
    return c[min(layer, len(c) - 1)]


def c_needed(got: torch.Tensor, want: torch.Tensor) -> float:
    """The smallest c for which err_ratios(got, want, c) <= 1 everywhere (rms over the last dimension)."""
    want = want.detach().double()
    got = got.detach().to(want.device, torch.float64).reshape(want.shape)
    rms = want.pow(2).mean(-1, keepdim=True).sqrt()
    need = ((got - want).abs() - ATTN_REL * want.abs()) / rms
    return float(torch.nan_to_num(need, nan=math.inf).max().clamp(min=0))


def dep_checkpoints(got: dict, want: dict) -> list[tuple[str, int, int | None, torch.Tensor, torch.Tensor]]:
    """Pairs up the checkpoints of one frame in the order the frame computes them: "din" of every sub-step, then per sub-step
    k the "k" and "v" of every layer and the "logits".  ``got`` holds the device's bf16 buffers in depformer_ref64's layout
    (din [B, dep_q, dd], k / v lists per layer of [B, H, dep_q, 64], logits [dep_q, B, card]).  Yields
    (kind, sub-step, layer or None, got, want) with the rms dimension last and the batch row first."""
    Q = want["logits"].shape[0]
    L = len(want["k"])
    out = [("din", k, None, got["din"][:, k], want["din"][:, k]) for k in range(Q)]
    for k in range(Q):
        for layer in range(L):
            out.append(("k", k, layer, got["k"][layer][:, :, k], want["k"][layer][:, :, k]))
            out.append(("v", k, layer, got["v"][layer][:, :, k], want["v"][layer][:, :, k]))
        out.append(("logits", k, None, got["logits"][k], want["logits"][k]))
    return out


def dep_c(kind: str, layer: int | None, int8: bool = False) -> float:
    if kind == "din":
        return DEP_C_DIN
    if kind == "logits":
        return DEP_C_LOGITS_I8 if int8 else DEP_C_LOGITS
    return dep_c_kv(layer, int8)


def dep_row_ratios(got: torch.Tensor, want: torch.Tensor, kind: str, layer: int | None, int8: bool = False) -> torch.Tensor:
    """Worst err_ratios of each batch row of one checkpoint under its constant (``int8``: the DEP_C_*_I8 constants): [B]
    (<= 1 passes)."""
    r = err_ratios(got, want, dep_c(kind, layer, int8))
    return r.reshape(r.shape[0], -1).amax(dim=1)


def dep_row_scaled(sd: dict, seed: int = 0) -> dict:
    """``sd`` with every row of each depformer linear (depformer_in, the in / out projections, gate / value, linear_out and the
    heads) multiplied by its own factor 2^u, u uniform in [-1, 1].  Synthetic uniform weights give every row the same absmax,
    hence the same int8 row scale in every linear and sub-step; trained weights do not.  On these weights a scale taken from
    the wrong row, half, linear or sub-step changes the int8 product."""
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    for n, t in sd.items():
        if n.startswith(("depformer_in.", "linears.")) or (n.startswith("depformer.layers.") and ".norm" not in n):
            f = torch.exp2(torch.empty(t.shape[0]).uniform_(-1, 1, generator=g)).to(t.device)
            out[n] = (t.float() * f[:, None]).to(t.dtype)
    return out


def exact_row_ratios(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """The verdict of a bit-exact checkpoint per batch row, on dep_row_ratios' scale: [B], 0 where the row equals bf16(want),
    1e9 where any element differs."""
    want = want.to(got.device).bfloat16()
    bad = got.reshape(got.shape[0], -1) != want.reshape(want.shape[0], -1)
    return bad.any(1).double().cpu() * 1e9


# Classifier-free guidance (lm.py:728-732, 828-833): the model runs 2B rows, rows [0, B) conditioned and [B, 2B) null, and the
# samplers read null + (cond - null) * coef.
def cfg_guide_bf16(model_logits: torch.Tensor, B: int, coef: float) -> torch.Tensor:
    """The guided logits as the reference computes them: three bf16 tensor operations on the model's bf16 logits [2B, card]
    (bf16(n + bf16(bf16(l - n) * coef))): [B, card] bf16, for bit-exact checks."""
    lg, null = model_logits[:B].bfloat16(), model_logits[B:2 * B].bfloat16()
    return null + (lg - null) * coef


def cfg_guide64(ref_logits: torch.Tensor, B: int, coef: float) -> torch.Tensor:
    """The same combination in float64, of a reference's float64 logits [2B, card]: [B, card]."""
    lg, null = ref_logits[:B].double(), ref_logits[B:2 * B].double()
    return null + (lg - null) * coef


# ---- fp64 reference of one Mimi streaming frame ----------------------------------------------------------------------------
# Acceptance rule of the Mimi checkpoints: |got - want| <= MIMI_REL |want| + c rms(want), the rms taken per (row, head) for the
# ring entries and per (row, checkpoint) for activations, one c per checkpoint kind (MIMI_C).  MIMI_REL is about eight fp32 ulps.
MIMI_REL = 2.0 ** -20


def rope_freqs64(D: int, max_period: float) -> torch.Tensor:
    """The fp32 RoPE frequencies of rope_ref (correctly rounded exp of the fp32 argument), as float64."""
    arg = torch.arange(D // 2, dtype=torch.float32) * torch.tensor(-math.log(max_period) * 2 / D, dtype=torch.float32)
    return torch.exp(arg.double()).float().double()


def device_rope_freqs(D: int, max_period: float) -> torch.Tensor:
    """The fp32 RoPE frequencies as the CUDA kernels compute them: CUDA's expf of the same fp32 argument, which is not always the
    correctly rounded value.  One ulp of a low frequency turns its pair by about 3e-3 rad at position 45 000, so a reference
    that must hold to fp32 rounding there has to use the kernel's frequencies.  Needs a GPU."""
    arg = torch.arange(D // 2, dtype=torch.float32) * torch.tensor(-math.log(max_period) * 2 / D, dtype=torch.float32)
    return torch.exp(arg.cuda()).cpu().double()


def rope64(x: torch.Tensor, pos: torch.Tensor, max_period: float, freqs: torch.Tensor | None = None) -> torch.Tensor:
    """Interleaved RoPE on [R, T, H, D] float64 at positions pos [R, T]: the angle is fp32(freq) * fp32(pos) rounded to fp32, as
    in rope_ref (freqs: fp32 values, rope_freqs64 by default); cos, sin and the rotation are float64."""
    R, T, H, D = x.shape
    f = (rope_freqs64(D, max_period) if freqs is None else freqs).float()
    ang = (f[None, None, :] * pos.float()[..., None]).double()                 # [R, T, D/2], fp32 product
    c, s = torch.cos(ang)[:, :, None], torch.sin(ang)[:, :, None]
    xr, xi = x[..., 0::2], x[..., 1::2]
    return torch.stack([xr * c - xi * s, xr * s + xi * c], dim=-1).reshape(R, T, H, D)


def ring_positions(off: torch.Tensor, T: int, cap: int, executing: torch.Tensor) -> torch.Tensor:
    """The absolute position held by every ring slot after a step of T tokens at offsets off [R] (RingKVCache.complete,
    transformer.py:236-288), -1 for an empty slot: [R, cap].  A paused row's ring is labelled as if it had appended (the kernel
    and the reference share this labelling); its offset does not move, so slots at and after it stay empty."""
    s = torch.arange(cap)
    last = off[:, None] + T - 1
    delta = s[None] - last % cap
    pos = torch.where(delta <= 0, last + delta, last + delta - cap)
    end = off[:, None] + T * executing.long()[:, None]
    return torch.where(s[None] >= end, torch.full_like(pos, -1), pos)


def attn_mask64(off: torch.Tensor, T: int, cap: int, context: int, executing: torch.Tensor, mutant: dict | None = None):
    """allowed [R, T, cap]: slot s may be attended by query t (transformer.py:576-580 with ring_positions).  Mutants:
    "drop_oldest" (each query loses its oldest allowed key), "q0_sees_q1" (query 0 also sees query 1's key)."""
    mutant = mutant or {}
    pk = ring_positions(off, T, cap, executing)[:, None, :]                    # [R, 1, cap]
    pq = (off[:, None] + torch.arange(T)[None])[..., None]                     # [R, T, 1]
    d = pq - pk
    allowed = (pk >= 0) & (d >= 0) & (d < context)
    if mutant.get("q0_sees_q1") and T > 1:
        allowed[:, 0] |= (pk[:, 0] == pq[:, 1])
    if mutant.get("drop_oldest"):
        oldest = torch.where(allowed, pk.expand_as(allowed), torch.full_like(allowed, 2 ** 62, dtype=torch.long)).amin(-1, keepdim=True)
        allowed &= pk != oldest
    return allowed


def ring_attention64(q: torch.Tensor, kring: torch.Tensor, vring: torch.Tensor, allowed: torch.Tensor) -> torch.Tensor:
    """softmax(q . k / 8) . v over the allowed slots in float64: q [R, T, H, D], rings [R, H, cap, D], allowed [R, T, cap]
    -> [R, T, H, D].  Masked slots are selected out (a NaN there cannot leak); a query with no key gives zeros."""
    s = torch.einsum("rthd,rhsd->rths", q.double(), torch.nan_to_num(kring.double())) * q.shape[-1] ** -0.5
    m = allowed[:, :, None, :]
    s = torch.where(m, s, torch.full_like(s, -math.inf))
    p = torch.softmax(s, dim=-1)
    p = torch.where(m, torch.nan_to_num(p), torch.zeros_like(p))
    return torch.einsum("rths,rhsd->rthd", p, torch.nan_to_num(vring.double()))


class MimiRef64:
    """One Mimi streaming frame (oracle/mimi.py's data path) in float64 for R selected sessions, teacher-forced stage by stage
    on the taps of the implementation under test, so that every kernel is judged alone and errors do not compound:

    * SEANet encoder / decoder: module i runs on the tap of module i - 1 (``taps``, the reference's names "enc.<i>" /
      "dec.<i>", [R, C, T]).  A streaming conv's carried left context is this object's own history of those taps (after the
      activation), a transposed conv's overlap-add carry this object's own partial: one source, the taps, for every carry.
    * bottleneck transformers: all 8 layers from the tap in front of them ("enc.14" / "dec.up"), attending over the rings the
      implementation held before the frame (``rings``: per layer (k, v) [R, H, cap, 64]) with the positions this object
      tracks.  Checkpoints: the new ring entries of every layer and the output ("enc.tr" / "dec.tr").
    * down-sampling conv from "enc.tr" (first-frame replicate padding), RVQ from the implementation's latent, residuals
      teacher-forced on its codes (level l searches the residual after the implementation's codes of levels < l).
    * decode: "dec.latent" from the implementation's codes, "dec.up" from its "dec.latent" with this object's overlap-add carry.

    Sessions are independent, so only the selected rows are computed.  ``exec`` is the exec_mask of those rows; ``reset(mask)``
    recycles rows like reset_streaming.

    ``mutant`` (for the tests of the acceptance rule) changes one thing:
      "weight": f(key, w) -> the tensor to use for state-dict key ``key``;
      "attn": dict with "drop_oldest" / "q0_sees_q1" / "overwritten" (query 0 also attends to the key this step overwrote);
      "rope_shift": added to every RoPE position;      "swap_layer_scales", "gelu_tanh", "ln_unbiased": True;
      "conv_shift": conv key whose carried context is committed one row early;   "no_elu": conv key fed without its ELU;
      "no_carry": key of a transposed conv whose overlap-add carry is dropped;
      "rvq_codebook_shift": (quantizer, level) searched with the next level's codebook;   "rvq_no_residual": True;
      "rvq_swap_proj": True (semantic and acoustic input projections swapped).
    ``rope_freqs``: the fp32 RoPE frequencies to use (rope_freqs64 by default; device_rope_freqs for a CUDA implementation)."""

    def __init__(self, sd: dict, cfg, R: int, mutant: dict | None = None, rope_freqs: torch.Tensor | None = None):
        from oracle.mimi import MimiOracle
        self.orc = MimiOracle(sd, cfg)
        self.freqs = rope_freqs
        self.cfg, self.R, self.mutant = cfg, R, mutant or {}
        self._w: dict = {}
        self.exec = torch.ones(R, dtype=torch.bool)
        self.prev: dict = {}
        self.part: dict = {}
        self.first = torch.ones(R, dtype=torch.bool)
        self.offset = {w: torch.zeros(R, dtype=torch.long) for w in ("encoder_transformer", "decoder_transformer")}

    def W(self, key: str) -> torch.Tensor | None:
        if key not in self._w:
            t = self.orc.sd.get(key)
            if t is not None:
                t = t.double()
                if "weight" in self.mutant:
                    t = self.mutant["weight"](key, t)
            self._w[key] = t
        return self._w[key]

    def reset(self, mask: torch.Tensor | None = None) -> None:
        mask = torch.ones(self.R, dtype=torch.bool) if mask is None else mask
        self.exec |= mask
        for t in list(self.prev.values()) + list(self.part.values()):
            t[mask] = 0
        self.first[mask] = True
        for off in self.offset.values():
            off[mask] = 0

    # ---- convolutions
    def _conv(self, spec, x: torch.Tensor) -> torch.Tensor:
        w, b = self.W(spec.key + ".weight"), self.W(spec.key + ".bias")
        P = (w.shape[-1] - 1) * spec.dilation + 1 - spec.stride
        m = self.exec.view(-1, 1, 1)
        if P == 0:
            return F.conv1d(x, w, b, stride=spec.stride, dilation=spec.dilation)
        st = self.prev.setdefault(spec.key, torch.zeros(self.R, x.shape[1], P, dtype=torch.float64))
        if spec.replicate:
            st = torch.where(self.first.view(-1, 1, 1) & m, x[..., :1].expand_as(st), st)
        xx = torch.cat([st, x], dim=-1)
        y = F.conv1d(xx, w, b, stride=spec.stride, dilation=spec.dilation)
        keep = xx[..., -P - 1:-1] if self.mutant.get("conv_shift") == spec.key else xx[..., -P:]
        self.prev[spec.key] = torch.where(m, keep, st)
        if spec.replicate:
            self.first &= ~self.exec
        return y

    def _convtr(self, spec, x: torch.Tensor) -> torch.Tensor:
        w, b = self.W(spec.key + ".weight"), self.W(spec.key + ".bias")
        K, S = w.shape[-1], spec.stride
        y = F.conv_transpose1d(x, w, b, stride=S, groups=spec.groups)
        pt = K - S
        part = self.part.setdefault(spec.key, torch.zeros(self.R, y.shape[1], pt, dtype=torch.float64))
        if self.mutant.get("no_carry") != spec.key:
            y[..., :pt] += part
        tail = y[..., -pt:] - (b[:, None] if b is not None else 0)
        self.part[spec.key] = torch.where(self.exec.view(-1, 1, 1), tail, part)
        return y[..., :-pt]

    def _act(self, key: str, x: torch.Tensor) -> torch.Tensor:
        return x if self.mutant.get("no_elu") == key else F.elu(x)

    def _seanet(self, plan: list, x: torch.Tensor, taps: dict, out: dict) -> None:
        for item in plan:
            if item[0] == "res":
                from oracle.mimi import ConvSpec
                _, base, dil = item
                k1, k3 = base + ".block.1.conv.conv", base + ".block.3.conv.conv"
                h = self._conv(ConvSpec(k1, "conv", dilation=dil), self._act(k1, x))
                y = x + self._conv(ConvSpec(k3, "conv"), self._act(k3, h))
                name = base
            else:
                spec = item[1]
                xin = self._act(spec.key, x) if spec.elu_before else x
                y = self._conv(spec, xin) if spec.kind == "conv" else self._convtr(spec, xin)
                name = spec.key
            side, _, idx = name.split(".")[:3]
            tap = f"{side[:3]}.{idx}"
            out[tap] = y
            x = taps[tap].double() if tap in taps else y

    # ---- transformer
    def _ln(self, x: torch.Tensor, p: str) -> torch.Tensor:
        mu = x.mean(-1, keepdim=True)
        var = (x - mu).pow(2).sum(-1, keepdim=True) / (x.shape[-1] - (1 if self.mutant.get("ln_unbiased") else 0))
        return (x - mu) / torch.sqrt(var + 1e-5) * self.W(p + ".weight") + self.W(p + ".bias")

    def _transformer(self, which: str, x: torch.Tensor, rings: list, out: dict) -> torch.Tensor:
        """x [R, T, C] float64 -> [R, T, C]; out gets "<which>.<l>.k" / ".v" [R, H, T, 64] (the entries this frame appends)."""
        cfg, mut = self.cfg, self.mutant
        R, T, C = x.shape
        H = cfg.tr_num_heads
        D = C // H
        off = self.offset[which]
        ex = self.exec
        pos = off[:, None] + torch.arange(T)[None] + mut.get("rope_shift", 0)
        am = mut.get("attn", {})
        allowed = attn_mask64(off, T, cfg.tr_context, cfg.tr_context, ex, am)
        slots = (off[:, None] + torch.arange(T)[None]) % cfg.tr_context
        ls1, ls2 = "layer_scale_1", "layer_scale_2"
        if mut.get("swap_layer_scales"):
            ls1, ls2 = ls2, ls1
        for li in range(cfg.tr_num_layers):
            p = f"{which}.transformer.layers.{li}"
            qkv = (self._ln(x, p + ".norm1") @ self.W(p + ".self_attn.in_projs.0.weight").T).view(R, T, 3, H, D)
            q, k, v = rope64(qkv[:, :, 0], pos, cfg.tr_max_period, self.freqs), rope64(qkv[:, :, 1], pos, cfg.tr_max_period, self.freqs), qkv[:, :, 2]
            kr, vr = rings[li][0].double().clone(), rings[li][1].double().clone()
            old_k, old_v = kr.clone(), vr.clone()
            for r in range(R):
                if ex[r]:
                    kr[r][:, slots[r]] = k[r].transpose(0, 1)
                    vr[r][:, slots[r]] = v[r].transpose(0, 1)
            o = ring_attention64(q, kr, vr, allowed)
            if am.get("overwritten"):
                # query 0 also attends to the key that slot (offset % cap) held before this step wrote it
                s0 = slots[:, 0]
                ko = torch.stack([old_k[r][:, s0[r]] for r in range(R)])[:, None]          # [R, 1, H, D]
                vo = torch.stack([old_v[r][:, s0[r]] for r in range(R)])[:, None]
                kk = torch.cat([kr, ko.permute(0, 2, 1, 3)], dim=2)
                vv = torch.cat([vr, vo.permute(0, 2, 1, 3)], dim=2)
                wrapped = (off >= cfg.tr_context)[:, None, None]
                al = torch.cat([allowed, wrapped.expand(R, T, 1) & (torch.arange(T) == 0)[None, :, None]], dim=2)
                o = ring_attention64(q, kk, vv, al)
            out[f"{which}.{li}.k"], out[f"{which}.{li}.v"] = k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)
            x = x + self.W(p + f".{ls1}.scale") * (o.reshape(R, T, C) @ self.W(p + ".self_attn.out_projs.0.weight").T)
            h = self._ln(x, p + ".norm2") @ self.W(p + ".linear1.weight").T
            h = F.gelu(h, approximate="tanh" if mut.get("gelu_tanh") else "none")
            x = x + self.W(p + f".{ls2}.scale") * (h @ self.W(p + ".linear2.weight").T)
        self.offset[which] = torch.where(ex, off + T, off)
        return x

    # ---- quantizer
    def _centroids(self, prefix: str) -> torch.Tensor:
        return self.W(prefix + ".embedding_sum") / self.W(prefix + ".cluster_usage").clamp(min=1e-5)[:, None]

    def quantize(self, latent: torch.Tensor, codes: torch.Tensor) -> dict:
        """latent [R, C] (the implementation's), codes [R, K] (its codes, which steer the residuals) -> "codes" [R, K] (fp64
        argmin, first index on ties), "gap" [R, K] (second-best minus best squared distance) and "scale" [R, K] (|r|^2 + |c|^2 of
        the best code: the size of the terms whose fp32 rounding can flip a near tie)."""
        mut = self.mutant
        n_sem = self.cfg.q_n_semantic
        K = codes.shape[1]
        names = [("rvq_first", 0, min(n_sem, K)), ("rvq_rest", min(n_sem, K), K)]
        proj = {n: f"quantizer.{n}.input_proj.weight" for n, _, _ in names}
        if mut.get("rvq_swap_proj"):
            proj = {"rvq_first": proj["rvq_rest"], "rvq_rest": proj["rvq_first"]}
        want = torch.zeros_like(codes)
        gap, scale = torch.zeros(codes.shape, dtype=torch.float64), torch.zeros(codes.shape, dtype=torch.float64)
        for name, lo, hi in names:
            if hi <= lo:
                continue
            res = latent.double() @ self.W(proj[name])[..., 0].T
            for level in range(hi - lo):
                lv = level + 1 if mut.get("rvq_codebook_shift") == (name, level) else level
                cb = self._centroids(f"quantizer.{name}.vq.layers.{lv}._codebook")
                d2 = (res[:, None, :] - cb[None]).pow(2).sum(-1)                   # [R, bins], exact enough in fp64
                two = torch.topk(d2, 2, dim=-1, largest=False)
                want[:, lo + level] = d2.argmin(-1)
                gap[:, lo + level] = two.values[:, 1] - two.values[:, 0]
                scale[:, lo + level] = res.pow(2).sum(-1) + cb[want[:, lo + level]].pow(2).sum(-1)
                if not mut.get("rvq_no_residual"):
                    res = res - self._centroids(f"quantizer.{name}.vq.layers.{level}._codebook")[codes[:, lo + level]]
        return dict(codes=want, gap=gap, scale=scale)

    def dequantize(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [R, K] -> latent [R, C, 1] (vq.py:281-287)."""
        n_sem, K = self.cfg.q_n_semantic, codes.shape[1]
        out = 0
        for name, lo, hi in (("rvq_first", 0, min(n_sem, K)), ("rvq_rest", min(n_sem, K), K)):
            if hi <= lo:
                continue
            q = sum(self._centroids(f"quantizer.{name}.vq.layers.{l}._codebook")[codes[:, lo + l]] for l in range(hi - lo))
            out = out + q @ self.W(f"quantizer.{name}.output_proj.weight")[..., 0].T
        return out[..., None]

    # ---- one frame
    def encode_frame(self, pcm: torch.Tensor, taps: dict, rings: list) -> dict:
        """pcm [R, 1, frame]; taps: the implementation's "enc.<i>", "enc.tr" [R, C, T] and "enc.latent" [R, C, 1]; rings:
        the encoder transformer's per-layer (k, v) before the frame.  Returns every checkpoint's float64 value."""
        out: dict = {}
        self._seanet(self.orc.enc_plan, pcm.double(), taps, out)
        last = [k for k in out if k.startswith("enc.")][-1]
        y = self._transformer("encoder_transformer", taps[last].double().transpose(1, 2), rings, out)
        out["enc.tr"] = y.transpose(1, 2)
        out["enc.latent"] = self._conv(self.orc.down_spec, taps["enc.tr"].double())
        return out

    def decode_frame(self, codes: torch.Tensor, taps: dict, rings: list) -> dict:
        """codes [R, K]; taps: "dec.latent" [R, C, 1], "dec.up" / "dec.tr" [R, C, T], "dec.<i>" (the last is the PCM)."""
        out = {"dec.latent": self.dequantize(codes)}
        out["dec.up"] = self._convtr(self.orc.up_spec, taps["dec.latent"].double())
        y = self._transformer("decoder_transformer", taps["dec.up"].double().transpose(1, 2), rings, out)
        out["dec.tr"] = y.transpose(1, 2)
        self._seanet(self.orc.dec_plan, taps["dec.tr"].double(), taps, out)
        return out


def mimi_kind(name: str, last_dec: str) -> str:
    """Checkpoint kind of a MimiRef64 checkpoint name."""
    if name.endswith((".k", ".v")):
        return "kv" + name.split(".")[-2]
    if name == last_dec:
        return "pcm"
    if name in ("enc.tr", "dec.tr", "enc.latent", "dec.latent", "dec.up"):
        return name
    return name[:3]


def mimi_ratios(got: torch.Tensor, want: torch.Tensor, c: float, per_head: bool = False) -> torch.Tensor:
    """Worst |got - want| / (MIMI_REL |want| + c rms) of each row: [R] (<= 1 passes).  The rms is over the row's whole
    checkpoint, or over each head ([R, H, ...] inputs) with ``per_head``."""
    want = want.detach().double()
    got = got.detach().double().reshape(want.shape)
    dims = tuple(range(2 if per_head else 1, want.dim()))
    rms = want.pow(2).mean(dim=dims, keepdim=True).sqrt()
    tol = MIMI_REL * want.abs() + c * rms
    r = torch.where(tol > 0, (got - want).abs() / tol, torch.where(got == want, 0.0, math.inf))
    r = torch.nan_to_num(r, nan=math.inf, posinf=math.inf)
    return r.reshape(r.shape[0], -1).amax(dim=1)


def mimi_c_needed(got: torch.Tensor, want: torch.Tensor, per_head: bool = False) -> float:
    want = want.detach().double()
    got = got.detach().double().reshape(want.shape)
    dims = tuple(range(2 if per_head else 1, want.dim()))
    rms = want.pow(2).mean(dim=dims, keepdim=True).sqrt()
    return float(torch.nan_to_num(((got - want).abs() - MIMI_REL * want.abs()) / rms, nan=math.inf).max().clamp(min=0))


# ---- fp64 reference of the temporal transformer, teacher-forced layer by layer -----------------------------------------------
def _tm_tensor(sd: dict, name: str, layer: int | None) -> torch.Tensor:
    """The state-dict tensor of the temporal transformer's weight ``name`` (at ``layer``); "din" is depformer_in.<layer>."""
    p = f"transformer.layers.{layer}."
    key = {"in": p + "self_attn.in_projs.0.weight", "out": p + "self_attn.out_projs.0.weight",
           "lin_in": p + "gating.linear_in.weight", "lin_out": p + "gating.linear_out.weight", "n1": p + "norm1.alpha",
           "n2": p + "norm2.alpha", "out_norm": "out_norm.alpha", "head": "text_linear.weight",
           "din": f"depformer_in.{layer}.weight", "cq": p + "cross_attention.in_projs.0.weight",
           "ckv": p + "cross_attention.in_projs.0.weight", "co": p + "cross_attention.out_projs.0.weight",
           "ncw": p + "norm_cross.weight", "ncb": p + "norm_cross.bias"}[name]
    if name in ("cq", "ckv"):       # transformer.py:495-505: rows [0, d) of in_projs.0 the query, [d, 3d) K|V of the condition
        d = sd[key].shape[1]
        return sd[key][:d] if name == "cq" else sd[key][d:]
    return sd[key]


def _tm_weights(sd: dict, layer: int | None, mutant: dict, dev):
    def W(name: str, at=layer) -> torch.Tensor:
        t = mutant["weight"](name, at, functools.partial(_tm_tensor, sd)) if "weight" in mutant else _tm_tensor(sd, name, at)
        return t.to(dev)
    return W


def _tm_linear(x: torch.Tensor, w: torch.Tensor, name: str, layer: int | None, quantize: bool, mutant: dict) -> torch.Tensor:
    """y = x . w^T in float64 for bf16-valued x, before the output's rounding; quantize: QLinear (oracle/quant.py: exact
    integer products, the fp32 dequantisation).  mutant["linear"](name, layer, x, w, y) -> y replaces the result."""
    if quantize:
        from oracle.quant import qlinear_f32
        y = qlinear_f32(x.to(torch.bfloat16), w).double()
    else:
        y = x.double() @ w.double().T
    return mutant["linear"](name, layer, x, w, y) if "linear" in mutant else y


def _tm_rmsnorm(x: torch.Tensor, alpha: torch.Tensor) -> torch.Tensor:
    """rmsnorm_ref64 on [R, dim] with the [1, 1, dim] alpha, not rounded."""
    x = x.double()
    return x * alpha.double().reshape(-1) / torch.sqrt(1e-8 + x.pow(2).mean(-1, keepdim=True))


def _res_add(cfg, layer: int, x: torch.Tensor, upd: torch.Tensor, which: str, mutant: dict) -> torch.Tensor:
    """x + upd of one residual (the fp32 add of the int8 epilogue under cfg.quantize); mutant["residual"] may drop it."""
    if not mutant.get("residual", lambda *a: True)(layer, which):
        return upd
    return (x.float() + upd.float()).double() if cfg.quantize else x.double() + upd


def _layernorm64(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """nn.LayerNorm over the last dimension in float64, not rounded."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = (x - mu).pow(2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w.double().reshape(-1) + b.double().reshape(-1)


def _softmax_attention64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, chunk: int = 16) -> torch.Tensor:
    """softmax(q . k_t / sqrt(D)) . v_t over every t, q [R, H, D], k / v [R, H, T, D] (any dtype) -> float64 [R, H, D], in
    chunks of rows on k's device (a memory of 625 keys at 512 rows is 5 GB in float64)."""
    R, H, D = q.shape
    out = []
    for i in range(0, R, chunk):
        kk, vv = k[i:i + chunk].double(), v[i:i + chunk].double()
        s = torch.einsum("rhd,rhtd->rht", q[i:i + chunk].to(kk.device, torch.float64), kk) * D ** -0.5
        out.append(torch.einsum("rht,rhtd->rhd", torch.softmax(s, dim=-1), vv))
        del kk, vv
    return torch.cat(out)


@torch.no_grad()
def cross_block_ref64(sd: dict, cfg, layer: int, x_attn: torch.Tensor, cross_out: torch.Tensor,
                      memory: tuple[torch.Tensor, torch.Tensor], mutant: dict | None = None) -> dict:
    """The cross-attention block of one temporal layer (transformer.py:779-798, tests/cross_oracle.py cross_block) in float64
    for R model rows, teacher-forced on the implementation's taps like temporal_layer_ref64:

      xn = bf16(layernorm(x_attn, norm_cross.weight, norm_cross.bias, eps 1e-5));  q = bf16(xn . in_projs.0[:d]^T);
      cross_out = softmax(q . k_t / sqrt(128)) . v_t over all T keys of the row's ``memory`` (the implementation's k_cross /
                  v_cross [R, H, T, 128]; no RoPE, no mask);
      x_cross = bf16(x_attn + bf16(out_projs.0(cross_out))).

    ``x_attn`` / ``cross_out`` are the implementation's x after the self-attention residual and its cross-attention output
    ([R, dim] bf16).  Returns, before their final bf16 rounding, as float64: "cross_out" [R, H, D], "x_cross" and the out
    linear's own output "x_cross.upd".  ``mutant`` as in temporal_layer_ref64 (weight / linear names cq, co, ncw, ncb;
    "residual" with "cross")."""
    mutant = mutant or {}
    dev = x_attn.device
    R, d = x_attn.shape
    H = cfg.num_heads
    W = _tm_weights(sd, layer, mutant, dev)
    xn = _bf(_layernorm64(x_attn, W("ncw"), W("ncb")))
    q = _bf(_tm_linear(xn, W("cq"), "cq", layer, False, mutant)).view(R, H, d // H)
    kx, vx = memory
    o = _softmax_attention64(q, kx, vx).to(dev)
    upd = _bf(_tm_linear(cross_out.double(), W("co"), "co", layer, False, mutant))
    return {"cross_out": o, "x_cross": _res_add(cfg, layer, x_attn, upd, "cross", mutant), "x_cross.upd": upd}


@torch.no_grad()
def cross_memory_ref64(sd: dict, cfg, layer: int, src: torch.Tensor, rows: int = 16):
    """The condition memory of one layer (transformer.py:495-505) in float64: k_cross | v_cross = src . in_projs.0[d:3d]^T
    split as "b t (p h d) -> p b h t d", for src [R, T, dim] bf16 (the fused condition, fuser.get_cross).  Yields (r0, k, v)
    per chunk of ``rows`` rows, k / v [n, H, T, 128] float64 before their bf16 rounding, on src's device: at R = 256 and
    T = 625 the whole product is 5 GB."""
    R, T, d = src.shape
    H = cfg.num_heads
    w = _tm_tensor(sd, "ckv", layer).to(src.device, torch.float64)
    for r0 in range(0, R, rows):
        kv = src[r0:r0 + rows].double() @ w.T
        kv = kv.view(-1, T, 2, H, d // H).permute(2, 0, 3, 1, 4)
        yield r0, kv[0], kv[1]
        del kv


@torch.no_grad()
def temporal_layer_ref64(sd: dict, cfg, layer: int, x_in: torch.Tensor, ao: torch.Tensor, x_attn: torch.Tensor, h: torch.Tensor,
                         kv_ring: tuple[torch.Tensor, torch.Tensor], pos: torch.Tensor, executing: torch.Tensor,
                         mutant: dict | None = None, rope_freqs: torch.Tensor | None = None, cross: dict | None = None) -> dict:
    """One temporal-transformer layer (transformer.py:752-802 with the gated SiLU of gating.py:13-22, as oracle/transformer.py
    states it) in float64 for R model rows, teacher-forced on the implementation's own taps so that each linear is judged on
    its own input and the error bound stays one cast point wide at every depth:

      xn = bf16(rmsnorm(x_in, norm1));  q, k, v = bf16(in_proj(xn));  k = RoPE(k, pos) (rope64);
      attn_out = softmax(q . k_j / sqrt(D)) . v_j over ``kv_ring`` (the implementation's rings after the step, [R, H, cap, D]),
                 with the reference's own rotated q (ring_attention64, attn_mask64 at ``pos`` / ``executing``);
      x_attn = bf16(x_in + bf16(out_proj(ao)));   gated = bf16(bf16(silu(bf16 g)) * bf16 u), g | u = linear_in(bf16 rmsnorm(x_attn));
      x_out = bf16(x_attn + bf16(linear_out(h))).

    ``x_in`` / ``ao`` / ``x_attn`` / ``h`` are the implementation's layer input and its attention output, x after the attention
    residual and gated hidden ([R, dim] / [R, ffn_hidden], bf16); ``pos`` [R] the positions before the step.  Runs on x_in's
    device, one layer's weights at a time.  Returns, before their final bf16 rounding, as float64: "k" / "v" [R, H, D] (the
    entry the step appends; only executing rows append), "attn_out" [R, H, D], "x_attn", "gated", "x_out", and the linears'
    own outputs "x_attn.upd" / "x_out.upd" (the residual checkpoints take their rms from these).  With cfg.quantize every linear
    is a QLinear and the residual adds are the fp32 adds of the int8 epilogue, so "x_attn" / "x_out" round to the exact bf16
    result given the taps.

    ``cross`` (a cross-attention layer): the implementation's "cross_out" and "x_cross" taps and its condition memory "kx" /
    "vx" [R, H, T, D].  The layer then also returns cross_block_ref64's "cross_out", "x_cross" and "x_cross.upd", and the MLP
    runs on the "x_cross" tap instead of x_attn: gated from rmsnorm(x_cross, norm2), x_out = x_cross + linear_out(h).

    ``mutant`` (for the tests of the acceptance rule) changes one thing:
      "weight": f(name, layer, fetch) -> the raw tensor (names in, out, lin_in, lin_out, n1, n2, and cq, co, ncw, ncb of the
                cross block; fetch(name, layer) is right);
      "linear": f(name, layer, x, w, y) -> the linear's float64 output y (x its input, w its weight);
      "residual": f(layer, "attn" | "cross" | "ffn") -> False to drop that residual;   "rope_shift": added to k's RoPE position."""
    mutant = mutant or {}
    dev = x_in.device
    R, d = x_in.shape
    H = cfg.num_heads
    D = d // H
    W = _tm_weights(sd, layer, mutant, dev)

    def lin(x, name):
        return _tm_linear(x, W(name), name, layer, cfg.quantize, mutant)

    def res_add(x, upd, which):
        return _res_add(cfg, layer, x, upd, which, mutant)

    qkv = lin(_bf(_tm_rmsnorm(x_in, W("n1"))), "in").view(R, 3, H, D)
    p = pos.cpu()
    q = rope64(_bf(qkv[:, 0]).cpu()[:, None], p[:, None], cfg.max_period, rope_freqs)
    k = rope64(_bf(qkv[:, 1]).cpu()[:, None], p[:, None] + mutant.get("rope_shift", 0), cfg.max_period, rope_freqs)[:, 0]
    kr, vr = kv_ring
    allowed = attn_mask64(p, 1, kr.shape[2], cfg.context, executing.cpu())
    o = torch.cat([ring_attention64(q[i:i + 16].to(dev), kr[i:i + 16], vr[i:i + 16], allowed[i:i + 16].to(dev))
                   for i in range(0, R, 16)])[:, 0]
    upd1 = _bf(lin(ao.double(), "out"))
    xa = res_add(x_in, upd1, "attn")
    out = {}
    x_mlp = x_attn
    if cross is not None:
        out = cross_block_ref64(sd, cfg, layer, x_attn, cross["cross_out"], (cross["kx"], cross["vx"]), mutant)
        x_mlp = cross["x_cross"]
    gu = lin(_bf(_tm_rmsnorm(x_mlp, W("n2"))), "lin_in")
    F_ = gu.shape[1] // 2
    g, u = _bf(gu[:, :F_]), _bf(gu[:, F_:])
    upd2 = _bf(lin(h.double(), "lin_out"))
    xo = res_add(x_mlp, upd2, "ffn")
    return {"k": k.to(dev), "v": qkv[:, 2], "attn_out": o, "x_attn": xa, "x_attn.upd": upd1, **out,
            "gated": _bf(g * torch.sigmoid(g)) * u, "x_out": xo, "x_out.upd": upd2}


@torch.no_grad()
def temporal_embed_ref64(sd: dict, cfg, input_tokens: torch.Tensor, condition_sum: torch.Tensor | None = None) -> torch.Tensor:
    """The summed input embeddings entering layer 0 (lm.py:379-399, lm_utils.py:102-124) in float64: text_emb of column 0 plus
    emb.<k> of column k + 1 of ``input_tokens`` [MB, n_q + 1] (the model rows' tokens, CFG rows included), token -1 -> the
    zero row, plus ``condition_sum`` [MB, dim] when given.  Exact: every term is bf16."""
    tok = input_tokens
    out = 0
    for k in range(tok.shape[1]):
        table = sd["text_emb.weight" if k == 0 else f"emb.{k - 1}.weight"]
        t = tok[:, k].to(table.device)
        out = out + table[t.clamp(min=0)].double() * (t >= 0)[:, None]
    if condition_sum is not None:
        out = out + condition_sum.double().to(out.device)
    return out


@torch.no_grad()
def temporal_embed_bf16(sd: dict, input_tokens: torch.Tensor, condition_sum: torch.Tensor | None = None) -> torch.Tensor:
    """The summed input embeddings as the bf16 model computes them (lm.py:390-399, oracle/lm.py forward_text): the audio tables
    emb.0 .. emb.<n_q - 1> in order, then text_emb, then ``condition_sum``, each add one bf16 tensor add (an fp32 sum rounded to
    bf16).  Every bf16 implementation that adds in this order gets these bits: [MB, dim] bf16."""
    tok = input_tokens
    x = None
    for k in list(range(1, tok.shape[1])) + [0]:
        table = sd["text_emb.weight" if k == 0 else f"emb.{k - 1}.weight"]
        t = tok[:, k].to(table.device)
        e = torch.where((t >= 0)[:, None], table[t.clamp(min=0)], torch.zeros((), dtype=table.dtype, device=table.device))
        x = e if x is None else x + e
    if condition_sum is not None:
        x = x + condition_sum.to(x.device, torch.bfloat16)
    return x


@torch.no_grad()
def temporal_heads_ref64(sd: dict, cfg, x_last: torch.Tensor, tout: torch.Tensor, mutant: dict | None = None) -> dict:
    """The heads of the temporal transformer in float64, teacher-forced: "transformer_out" = rmsnorm(``x_last``, out_norm) (the
    implementation's x after the last layer), "text_logits" [MB, text_card] and "dep_in" [MB, dep_q, depformer_dim]
    (depformer_in[k] for every k, which the implementation writes as one [MB, dep_q * dd] product) of its ``tout``, all before
    their final rounding; with extra heads (the STT models) also "extra_heads" (extra_heads_ref64).  ``mutant``: "weight" /
    "linear" as in temporal_layer_ref64 (names out_norm, head, din; din's layer is the sub-step k); it does not reach the
    extra heads, whose mutants extra_heads_ref64 takes in its own form."""
    mutant = mutant or {}
    dev = tout.device
    W = _tm_weights(sd, None, mutant, dev)
    out = {"transformer_out": _tm_rmsnorm(x_last, W("out_norm")),
           "text_logits": _tm_linear(tout.double(), W("head"), "head", None, cfg.quantize, mutant)}
    if cfg.dep_q > 0:
        out["dep_in"] = torch.stack([_tm_linear(tout.double(), W("din", k), "din", k, cfg.quantize, mutant)
                                     for k in range(cfg.dep_q)], dim=1)
    if cfg.extra_heads_num_heads > 0:
        out["extra_heads"] = extra_heads_ref64(sd, cfg, tout)
    return out


# ---- the extra heads of the STT models ---------------------------------------------------------------------------------------
@torch.no_grad()
def extra_heads_ref64(sd: dict, cfg, tout: torch.Tensor, mutant: dict | None = None) -> dict:
    """softmax(extra_heads.<i>(transformer_out)) of every head (lm.py:224-226, 803-806) in float64, teacher-forced on the
    implementation's ``tout`` [MB, dim] bf16: the logits tout . w_i^T in float64 rounded to bf16 (nn.Linear's output is a bf16
    tensor), then a float64 softmax over the E = extra_heads_dim logits of the head.  Returns "logits" [n, MB, E] (bf16-valued)
    and "p" [n, MB, E], the probabilities before their bf16 rounding.

    ``mutant`` (for the tests of the rule): "weight": f(i, fetch) -> head i's [E, dim] weight (fetch(i) is right);
    "logits": f(logits [n, MB, E] float64 before rounding) -> the logits the softmax of each head runs over (may add entries)."""
    mutant = mutant or {}
    n = cfg.extra_heads_num_heads

    def fetch(i):
        return sd[f"extra_heads.{i}.weight"]
    x = tout.double()
    w = [(mutant["weight"](i, fetch) if "weight" in mutant else fetch(i)).to(x.device, torch.float64) for i in range(n)]
    lg = torch.stack([x @ wi.T for wi in w])
    if "logits" in mutant:
        lg = mutant["logits"](lg)
    lg = _bf(lg)
    return {"logits": lg[..., :cfg.extra_heads_dim], "p": torch.softmax(lg, dim=-1)[..., :cfg.extra_heads_dim]}


def _bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """The spacing of bf16 numbers just above |x| (float64; the smallest normal's spacing at 0)."""
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 7)


def extra_heads_ratios(got: torch.Tensor, ref: dict) -> torch.Tensor:
    """Worst |got - p| / tol of each (head, row) of the extra heads' probabilities ``got`` [n, MB, E] (bf16): [n, MB], <= 1
    passes.  The implementation's bf16 logit may land one bf16 ulp u_j away from the reference's (an fp32 sum in another order
    near a rounding boundary), which moves p_i by at most p_i (u_i + sum_j p_j u_j) to first order; its fp32 softmax adds a
    relative 2^-16 and the bf16 rounding of the probability half an ulp of p:
        tol_i = 1.25 p_i (u_i + sum_j p_j u_j) + 2^-16 p_i + ulp(p_i) / 2."""
    p, u = ref["p"], _bf16_ulp(ref["logits"])
    got = got.to(p.device, torch.float64).reshape(p.shape)
    tol = 1.25 * p * (u + (p * u).sum(-1, keepdim=True)) + 2.0 ** -16 * p + 0.5 * _bf16_ulp(p)
    r = torch.nan_to_num((got - p).abs() / tol, nan=math.inf, posinf=math.inf)
    return r.amax(-1)


# Acceptance rule of the temporal checkpoints: |got - want| <= TM_REL |want| + c rms, one c per checkpoint kind for every layer.
# The rms is taken per (row, head) for k, v and attn_out, per row of the checkpoint for embed, gated, transformer_out,
# text_logits and dep_in (per sub-step), and for the residual checkpoints x_attn / x_out per row of the linear's own output
# (".upd"): a large residual must not hide a lost k-block.  Each c is about twice what the bf16 oracle (oracle/lm.py) needs
# against the references at the 7B layer shapes (2 layers, two steps, rings of history; tests/test_temporal_ref_cpu.py
# measures it again and asserts that the oracle passes).  What it needs at B = 4 / B = 256:
#   embed 0.024 / 0.043 (the oracle adds the 17 embeddings in bf16, one rounding per add), k 0.0012 / 0.0073,
#   v 1.8e-8 / 4.4e-4, attn_out 0.0092 / 0.013, x_attn 0.0020 / 0.0070, gated 1.4e-5 / 0.037, x_out 0 / 0.0048,
#   transformer_out 0 / 0, text_logits 1.6e-7 / 4.4e-7, dep_in 0 / 4.4e-7.
# B = 256 samples the rare rounding flips (a gate input one ulp off moves silu(g) u by far more than its rms share) that four
# rows miss, so it sets the constants.  transformer_out and the heads need nothing beyond the relative term: they get a floor
# of 2^-10 for fp32 accumulation in another order.
# At the 2B shapes (tests/golden/moshi_dev_2b.json: dim 2560, 20 heads, ffn 7040, RoPE period 1e5, 33 embedding tables and a
# condition sum, text_card 48000, depformer_in 16 x 1024; two layers, B = 4 / 256, the same test file) the oracle needs:
#   embed 0.010 / 0.013, k 1.6e-6 / 0.0124, v 0 / 5.9e-4, attn_out 0.0081 / 0.012, x_attn 0 / 0.0042, gated 1.6e-4 / 0.014,
#   x_out 0 / 0.012, transformer_out 0 / 0, text_logits 8.3e-9 / 3.7e-7, dep_in 7.9e-9 / 2.8e-7.
# k (0.015 from the 7B shapes, 1.2 times that) gets 0.025; the k mutants need at least 0.48 at either geometry.  How much of
# embed's constant a correct sum needs depends on the tables' values: on tiled_lm_state_dict weights with a condition sum the
# handle's sum, bit-exact to the reference's order of bf16 adds, reached 0.83 of it.  tests/test_gpu_zz_temporal_ref.py
# therefore holds the embeddings bit for bit to temporal_embed_bf16, which every bf16 implementation in that order computes.
# Three kinds are set from what the handle needs instead (tests/test_gpu_zz_temporal_ref.py over all its cases, one H100 80GB
# HBM3, power limit 700 W), because the handle samples the same rare flips over far more rows and layers than the oracle:
#   x_attn 0.017 and x_out 0.013: the update's own bf16 rounding may land one ulp away from the reference's (fp32 sums in
#     another order), which at an update element of 4-5 rms is 0.016-0.02 of the rms; they get 0.035 and 0.03;
#   gated 0.076 (the 32-layer model) gets 0.15;   v 0.0015 (int8: one int8 step of an activation that sits on a rounding
#     boundary of the quantiser moves the whole row's product) gets 0.003.
# The mutants of tests/test_temporal_ref_cpu.py need at least 0.41 at x_attn / x_out and 3.3 at gated: still far outside.
# Cross-attention layers add four kinds, calibrated by tests/test_cross_ref_cpu.py on the bf16 cross oracle (dim 2048, 16
# heads, T = 125 condition keys, B = 4 / 256):
#   kx / vx, the condition memory with the rms per (row, head, key), need 4.7e-7 (one bf16 rounding of an fp32 product,
#     inside the relative term) and get the floor 2^-10;   cross_out (rms per row and head) needs 0.0031 and gets 0.008;
#   x_cross needs 0.0022 from the oracle but about 0.017 on the handle (tests/test_gpu_zz_cross_ref.py over all its cases, one
#     H100 80GB HBM3, power limit 700 W: the update's own rounding one ulp away, as at x_attn) and gets x_attn's 0.035.
# The cross mutants need at least 0.13 at cross_out, 0.86 at x_cross and 1.5 at kx.
TM_REL = 2.0 ** -7
TM_C = {"embed": 0.09, "k": 0.025, "v": 0.003, "attn_out": 0.027, "x_attn": 0.035, "gated": 0.15, "x_out": 0.03,
        "transformer_out": 2.0 ** -10, "text_logits": 2.0 ** -10, "dep_in": 2.0 ** -10,
        "kx": 2.0 ** -10, "vx": 2.0 ** -10, "cross_out": 0.008, "x_cross": 0.035}
TM_KINDS = tuple(TM_C)


def tm_row_ratios(got: torch.Tensor, want: torch.Tensor, kind: str, scale: torch.Tensor | None = None,
                  c: float | None = None) -> torch.Tensor:
    """Worst |got - want| / (TM_REL |want| + c rms) of each row: [R] (<= 1 passes).  The rms is over the last dimension of
    ``scale`` (default ``want``); a NaN never passes."""
    want = want.detach().double()
    got = got.detach().to(want.device, torch.float64).reshape(want.shape)
    s = (want if scale is None else scale.detach().to(want.device, torch.float64).reshape(want.shape)).pow(2)
    tol = TM_REL * want.abs() + (TM_C[kind] if c is None else c) * s.mean(-1, keepdim=True).sqrt()
    r = torch.where(tol > 0, (got - want).abs() / tol, torch.where(got == want, 0.0, math.inf))
    r = torch.nan_to_num(r, nan=math.inf, posinf=math.inf)
    return r.reshape(r.shape[0], -1).amax(dim=1)


def tm_c_needed(got: torch.Tensor, want: torch.Tensor, scale: torch.Tensor | None = None) -> float:
    """The smallest c for which tm_row_ratios passes everywhere."""
    want = want.detach().double()
    got = got.detach().to(want.device, torch.float64).reshape(want.shape)
    s = (want if scale is None else scale.detach().to(want.device, torch.float64).reshape(want.shape))
    rms = s.pow(2).mean(-1, keepdim=True).sqrt()
    return float(torch.nan_to_num(((got - want).abs() - TM_REL * want.abs()) / rms, nan=math.inf).max().clamp(min=0))


def tm_layer_checkpoints(want: dict, got: dict, rows: torch.Tensor) -> list[tuple[str, torch.Tensor, torch.Tensor, torch.Tensor | None]]:
    """(kind, got, want, rms source) of one layer in the order the layer computes them, the rms dimension last.  ``got`` holds
    the implementation's "k" / "v" [R, H, D] (its ring entries at the step's slot), "attn_out", "x_attn", "gated", "x_out",
    and on a cross-attention layer (``want`` from temporal_layer_ref64 with ``cross``) "cross_out" and "x_cross" between
    x_attn and gated; ``rows`` selects the executing rows for k and v (only they append)."""
    R = want["attn_out"].shape[0]
    H, D = want["attn_out"].shape[1:]
    cross = [("cross_out", got["cross_out"].reshape(R, H, D), want["cross_out"], None),
             ("x_cross", got["x_cross"], want["x_cross"], want["x_cross.upd"])] if "cross_out" in want else []
    return [("k", got["k"][rows], want["k"][rows], None), ("v", got["v"][rows], want["v"][rows], None),
            ("attn_out", got["attn_out"].reshape(R, H, D), want["attn_out"], None),
            ("x_attn", got["x_attn"], want["x_attn"], want["x_attn.upd"]), *cross,
            ("gated", got["gated"], want["gated"], None),
            ("x_out", got["x_out"], want["x_out"], want["x_out.upd"])]


def rvq_unexcused(got: torch.Tensor, ref: dict, bound: float) -> torch.Tensor:
    """[R, K] bool: device code differs from the fp64 code although the fp64 gap exceeds bound * scale."""
    return (got.cpu() != ref["codes"]) & (ref["gap"] > bound * ref["scale"])


# One constant per checkpoint kind: about twice what the fp32 CPU oracle (oracle/mimi.py) needs against MimiRef64 over 4
# sessions, 2 fresh frames and 3 frames across the ring wrap (tests/test_mimi_ref_cpu.py measures it again, prints both and
# asserts that the oracle passes).  What the oracle needs: SEANet encoder taps 2.0e-6, decoder taps 3.5e-6, PCM 5.3e-7,
# transformer outputs 8.3e-7 (encoder) and 7.1e-7 (decoder), latent 6.2e-7, dequantised latent 1.0e-6, up-sampled 9.1e-8, ring
# entries of layers 0..7 between 3.9e-6 and 5.8e-6.  The ring entries do not grow with depth here: each layer starts from a
# LayerNorm, and the largest share comes from the oracle's RoPE (one frequency one fp32 ulp off) at the wrapped offsets, which
# is the same in every layer; they share one constant.
MIMI_C = {"enc": 4e-6, "dec": 7e-6, "pcm": 1.1e-6, "enc.tr": 1.7e-6, "dec.tr": 1.4e-6, "enc.latent": 1.2e-6, "dec.latent": 2e-6,
          "dec.up": 2e-7, **{f"kv{l}": 1.2e-5 for l in range(8)}}

# The handle's kernels: the SEANet layers, the transformer linears and the decoder's last conv run 3xTF32 on the tensor cores
# (hi / lo split of both operands, the lo * lo product dropped: about 2^-22 per product instead of fp32's 2^-24), with long
# reductions (up to 16 384 terms) in one fp32 chain at large batch.  Judged under MIMI_C over every case of
# tests/test_gpu_zz_mimi_ref.py on one H100 80GB HBM3 (power limit 700 W), the handle needed up to 7.2 times MIMI_C on the
# encoder taps, 4.5 times on the decoder taps, 3.7 times on the transformer outputs and 1.2 times on the PCM; the ring entries,
# latents and the up-sampling stayed under 0.75 times MIMI_C.  Those four kinds get about twice the measured need; the rest keep the fp32 oracle's constants.
MIMI_C_TC = {**MIMI_C, "enc": 6e-5, "dec": 6e-5, "enc.tr": 1.2e-5, "dec.tr": 1.2e-5, "pcm": 2.5e-6}
# Those constants hold while no SEANet layer of the side accumulates more than MIMI_TC_CHAIN k-blocks in one chain (the longest
# chain up to 256 sessions at 132 SMs: encoder.6's 40).  From 257 sessions the plan stops splitting encoder.9 (96 k-blocks)
# and decoder.1 (64), whose tensor-core accumulation then errs more (tc_c); on one H100 80GB HBM3 (power limit 700 W) the
# encoder taps needed 1.69 times MIMI_C_TC there and the decoder taps 1.21 times.  The "enc" / "dec" constants grow in
# proportion to the side's longest chain beyond MIMI_TC_CHAIN (mimi_tc_chain_factor).
MIMI_TC_CHAIN = 40


def mimi_tc_chain_factor(lib, sms: int, B: int, side: str) -> float:
    """max(1, longest k-blocks per split of the ``side`` ("encoder" / "decoder") SEANet layers at B sessions / MIMI_TC_CHAIN)."""
    t = mimi_plan_runs(lib, sms)
    chain = max(next(f[3] for b0, b1, f in runs if b0 <= B <= b1) for n, runs in t["runs"].items() if n.startswith(side + "."))
    return max(1.0, chain / MIMI_TC_CHAIN)

# A device code may differ from the fp64 code only where the fp64 gap between the best and the second-best squared distance
# is at most RVQ_GAP_BOUND (|r|^2 + |c|^2): the fp32 search forms |c|^2 - 2 r.c over 256 products, whose rounding is below
# 256 * 2^-24 * 2 |r| |c| <= 2^-15 (|r|^2 + |c|^2) per code.
RVQ_GAP_BOUND = 2.0 ** -15


def mimi_checkpoints(want: dict, taps: dict, rings_after: dict, off_before: dict, executing: torch.Tensor, cap: int) -> list:
    """Tuples (name, got, want, per_head) of one frame, in the order the frame computes them.  ``taps`` are the
    implementation's activations in the reference layout; ``rings_after`` maps "<which>.<l>.k" / ".v" to its ring
    [R, H, cap, 64] after the frame; the new entries are taken from slots (offset + t) % cap of the executing rows (a paused
    row's ring is checked elsewhere: it must not change)."""
    out = []
    for name, w in want.items():
        if name.endswith((".k", ".v")):
            which = name.split(".")[0]
            T = w.shape[2]
            slots = (off_before[which][:, None] + torch.arange(T)[None]) % cap                 # [R, T]
            ring = rings_after[name]
            g = torch.stack([ring[r][:, slots[r]] for r in range(ring.shape[0])])
            rows = executing.nonzero().flatten()
            out.append((name, g[rows], w[rows], True))
        else:
            out.append((name, taps[name], w, False))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The Exp(1) noise the LM step draws itself (lm_noise_kernel, csrc/lm_kernels.cuh)
# ---------------------------------------------------------------------------------------------------------------------------
_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC 2011; the Random123 reference): ``ctr`` [..., 4] and ``key`` [..., 2] 32-bit words
    (broadcast against each other) -> [..., 4] uint32.  Every product is formed exactly in uint64."""
    c = np.asarray(ctr, dtype=np.uint64) & _U32
    k = np.asarray(key, dtype=np.uint64) & _U32
    c0, c1, c2, c3 = c[..., 0], c[..., 1], c[..., 2], c[..., 3]
    k0, k1 = k[..., 0], k[..., 1]
    m0, m1 = np.uint64(_PHILOX_M[0]), np.uint64(_PHILOX_M[1])
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _U32)
        k0 = (k0 + np.uint64(_PHILOX_W[0])) & _U32
        k1 = (k1 + np.uint64(_PHILOX_W[1])) & _U32
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def step_words(seed: int, ctr: int, n: int) -> np.ndarray:
    """The n raw 32-bit words of one step: element i is word i % 4 of Philox block q = i // 4, with counter
    (q low, q high, ctr low, ctr high) and key (seed low, seed high)."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    c = np.stack([q & _U32, q >> np.uint64(32), np.full_like(q, ctr & 0xFFFFFFFF), np.full_like(q, (ctr >> 32) & 0xFFFFFFFF)], -1)
    return philox4x32_10(c, np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64)).reshape(-1)[:n]


def exp1_ref64(m: np.ndarray) -> np.ndarray:
    """fp64 -log((m + 1) / 2^24) of 24-bit patterns m."""
    return -np.log((np.asarray(m, dtype=np.float64) + 1.0) / 2.0 ** 24)


def step_noise_ref(seed: int, ctr: int, n: int) -> tuple[np.ndarray, np.ndarray]:
    """(24-bit patterns r >> 8 as uint32, fp64 Exp(1) draws) of the n noise elements of step ``ctr`` under ``seed``."""
    m = step_words(seed, ctr, n) >> np.uint32(8)
    return m, exp1_ref64(m)


def f32_ulp(x: np.ndarray) -> np.ndarray:
    """One fp32 ulp at |x| (the spacing above |x| rounded to fp32)."""
    a = np.abs(np.asarray(x, dtype=np.float32))
    return (np.nextafter(a, np.float32(np.inf)) - a).astype(np.float64)


# ---- the plans of the LM's linears and of the fused depformer, as runs of batch sizes ------------------------------------------
LINEAR_PLAN_FIELDS = ["kernel", "m0", "rows", "grid", "cluster", "smem", "stages", "stage_bytes", "np", "Mpad", "kb_per", "S", "kbps",
                      "unit_tiles", "ldw", "Wc", "whole_rounds", "sk_tile0", "sk_items"]
LINEAR_KERNELS = {1: "gemv", 2: "ns", 3: "cluster-sk", 4: "stream-k"}
DEPFORMER_PHASES = ["in_proj", "out_proj", "linear_in", "linear_out", "head"]
DEPFORMER_PLAN_FIELDS = ["path", "part_floats", "stages", "stage_bytes", "smem", "grid"] + [
    f"{p}.{f}" for p in DEPFORMER_PHASES for f in ("n_tiles", "num_kb", "kbps", "S", "A", "N")]


def linear_plan(lib, M: int, N: int, K: int, epi: int, gate_rows: int, norm: int, int8: int, sms: int,
                gemv_max_rows: int) -> tuple[int, list[list[int]]]:
    """(norm folded, launches) of b200_op_linear_plan: LINEAR_PLAN_FIELDS per launch."""
    from moshi_b200 import _lib
    n = len(LINEAR_PLAN_FIELDS)
    cap = 2 + 4 * n
    buf = (C.c_int64 * cap)()
    rc = lib.b200_op_linear_plan(M, N, K, epi, gate_rows, int8, norm, sms, gemv_max_rows, buf, cap)
    assert rc == _lib.B200_OK, (M, N, K, epi, gate_rows, norm, int8, sms, gemv_max_rows, rc)
    return int(buf[1]), [list(buf[2 + n * i:2 + n * (i + 1)]) for i in range(int(buf[0]))]


def linear_plan_runs(lib, N: int, K: int, epi: int, gate_rows: int, norm: int, int8: int, sms: int, gemv_max_rows: int,
                     max_m: int = 256) -> list[tuple[int, int, list[list[int]]]]:
    """The batch sizes 1..max_m of one linear grouped into runs (first M, last M, launches of the first M) of equal plans, as
    tools/gen_linear_plans.py compresses them: within a run the launches are the same except for the row count of the last."""
    rows = LINEAR_PLAN_FIELDS.index("rows")
    runs: list[list] = []
    for M in range(1, max_m + 1):
        folded, blocks = linear_plan(lib, M, N, K, epi, gate_rows, norm, int8, sms, gemv_max_rows)
        if runs:
            first, _, f0, b0 = runs[-1]
            grown = [list(b) for b in b0]
            grown[-1][rows] += M - first
            if f0 == folded and grown == blocks:
                runs[-1][1] = M
                continue
        runs.append([M, M, folded, blocks])
    return [(first, last, blocks) for first, last, _, blocks in runs]


def depformer_plan(lib, geom, B: int, cfg: int, int8: int, mode: int, sms: int, gemv_max_rows: int) -> list[int]:
    """b200_op_depformer_plan for `geom` = (dep_q, depformer_dim, heads, ffn, card): DEPFORMER_PLAN_FIELDS."""
    from moshi_b200 import _lib
    n = len(DEPFORMER_PLAN_FIELDS)
    buf = (C.c_int64 * n)()
    rc = lib.b200_op_depformer_plan(*geom, B, cfg, int8, mode, sms, gemv_max_rows, buf, n)
    assert rc == _lib.B200_OK, (geom, B, cfg, int8, mode, sms, gemv_max_rows, rc)
    return list(buf)


def depformer_plan_runs(lib, geom, cfg: int, int8: int, mode: int, sms: int, gemv_max_rows: int,
                        max_b: int = 256) -> list[tuple[int, int, list[int]]]:
    """The sessions 1..max_b (1..max_b / 2 under guidance) grouped into runs (first B, last B, plan of the first B) of equal
    depformer plans, as tools/gen_depformer_plans.py compresses them: within a run only the partial-buffer floats change, in
    proportion to B."""
    runs: list[list] = []
    for B in range(1, (max_b // 2 if cfg else max_b) + 1):
        p = depformer_plan(lib, geom, B, cfg, int8, mode, sms, gemv_max_rows)
        if runs:
            first, _, p0 = runs[-1]
            grown = list(p0)
            grown[1] = p0[1] // first * B
            if grown == p:
                runs[-1][1] = B
                continue
        runs.append([B, B, p])
    return [tuple(r) for r in runs]


# ---- one linear against fp64 -----------------------------------------------------------------------------------------------
# Acceptance rule of one LM linear y = epi(x . W^T) (bf16 operands, fp32 accumulation): y must be a faithful bf16 rounding of
# the fp64 reference, where the product may be off by LINEAR_C * 2^-24 * sum_k |x_k w_k| (an fp32 sum in another order; it only
# decides near-zero outputs and rounding boundaries), every intermediate the epilogue rounds to bf16 (the residual add's
# update, the gated MLP's gate and value, the RMSNorm output folded into the GEMV) may be either faithful rounding of its
# reference, and silu one bf16 ulp off (or -0 where fp32's exp(-g) overflows).  A lost or doubled k-block, a lost K tail of 8 columns, a partial added twice, a wrong
# row or a wrong weight tile moves outputs by many ulps: tests/test_plan_runs_cpu.py shows that the rule rejects each of them.
# On one H100 every linear plan of tests/test_gpu_zz_plan_runs.py needed LINEAR_C of at most 4.
STORE, RESADD, GATE = 0, 1, 2
LINEAR_C = 32.0
# the RMSNorm the GEMV folds in is fp32: where fp64 puts an element within NORM_BAND (relative) of a bf16 midpoint, the kernel
# may round it the other way
NORM_BAND = 2.0 ** -16
_SILU_ARGMIN = -1.2784645427610738


def _bf_grid(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers in the binade of each |v| (float64; 2^-133 below the smallest normal)."""
    _, e = torch.frexp(v)
    return torch.ldexp(torch.ones_like(v), (e - 8).clamp(min=-133))


def bf_floor(v: torch.Tensor) -> torch.Tensor:
    """The largest bf16 number <= v (float64 in, float64 out)."""
    sp = _bf_grid(v)
    return torch.floor(v / sp) * sp


def bf_ceil(v: torch.Tensor) -> torch.Tensor:
    """The smallest bf16 number >= v (float64 in, float64 out)."""
    sp = _bf_grid(v)
    return torch.ceil(v / sp) * sp


def bf_next_up(v: torch.Tensor) -> torch.Tensor:
    """The bf16 number after the bf16 number v (float64)."""
    m, e = torch.frexp(v)
    sp = torch.ldexp(torch.ones_like(v), (e - 8).clamp(min=-133))
    sp = torch.where(m == -0.5, sp / 2, sp)              # from -2^k up: the spacing of the binade below 2^k
    return torch.where(v == 0, torch.full_like(v, 2.0 ** -133), v + sp)


def bf_next_down(v: torch.Tensor) -> torch.Tensor:
    return -bf_next_up(-v)


def _silu64(v: torch.Tensor) -> torch.Tensor:
    return v / (1.0 + torch.exp(-v))


def linear_ref64(x: torch.Tensor, w: torch.Tensor, epi: int = STORE, gate_rows: int = 0, res: torch.Tensor | None = None,
                 alpha: torch.Tensor | None = None) -> dict:
    """fp64 reference of y = epi(x . w^T) (w [N, K], gated: rows gate | value) on the operands' device: the product ``acc``,
    ``mag`` = sum_k |x_k w_k|, and, with ``alpha``, the product of bf16(rmsnorm_ref64(x, alpha)) plus in ``norm_slack`` what
    rounding its elements within NORM_BAND of a midpoint the other way can move it."""
    xd = x.double()
    wd, wa = w.double(), w.double().abs()
    norm_slack = None
    if alpha is not None:
        xn = rmsnorm_ref64(x, alpha)
        xd = _bf(xn)
        norm_slack = (_bf(xn * (1 + NORM_BAND)) - _bf(xn * (1 - NORM_BAND))).abs() @ wa.t()
    return dict(acc=xd @ wd.t(), mag=xd.abs() @ wa.t(), norm_slack=norm_slack, epi=epi, gate_rows=gate_rows,
                res=None if res is None else res.to(xd.device, torch.float64))


def linear_bounds(ref: dict, c: float = LINEAR_C) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(lowest, highest, nominal) output the rule of LINEAR_C accepts, per element (float64)."""
    acc = ref["acc"]
    s = c * 2.0 ** -24 * ref["mag"]
    if ref["norm_slack"] is not None:
        s = s + ref["norm_slack"]
    t_lo, t_hi = bf_floor(acc - s), bf_ceil(acc + s)
    if ref["epi"] == STORE:
        return t_lo, t_hi, acc
    if ref["epi"] == RESADD:
        r = ref["res"]
        return bf_floor(r + t_lo), bf_ceil(r + t_hi), r + _bf(acc)
    H = ref["gate_rows"]
    g_lo, g_hi, u_lo, u_hi = t_lo[:, :H], t_hi[:, :H], t_lo[:, H:], t_hi[:, H:]
    a, b = _silu64(g_lo), _silu64(g_hi)
    s_lo = torch.minimum(a, b)
    s_lo = torch.where((g_lo <= _SILU_ARGMIN) & (g_hi >= _SILU_ARGMIN), _silu64(torch.full_like(s_lo, _SILU_ARGMIN)), s_lo)
    s_hi = torch.maximum(a, b)
    # an fp32 silu g / (1 + exp(-g)) is -0 once exp(-g) overflows (g < -88.7, where silu > -2^-121)
    s_hi = torch.where(s_lo > -2.0 ** -100, s_hi.clamp(min=0.0), s_hi)
    s_lo, s_hi = bf_next_down(bf_floor(s_lo)), bf_next_up(bf_ceil(s_hi))        # silu one bf16 ulp off
    corners = torch.stack([s_lo * u_lo, s_lo * u_hi, s_hi * u_lo, s_hi * u_hi])
    nominal = _bf(_silu64(_bf(acc[:, :H]))) * _bf(acc[:, H:])
    return bf_floor(corners.amin(0)), bf_ceil(corners.amax(0)), nominal


def linear_ratios(y: torch.Tensor, ref: dict, c: float = LINEAR_C) -> torch.Tensor:
    """Per output element, how far y sits from the nominal reference toward the bound the rule accepts on its side (<= 1
    passes; a NaN never does).  A faithful rounding on the far side of the reference sits on that bound and scores exactly 1,
    so past pass / fail the ratio says little; linear_c_needed grades a passing output."""
    lo, hi, nom = linear_bounds(ref, c)
    y = y.detach().to(nom.device, torch.float64).reshape(nom.shape)
    r = torch.where(y > nom, (y - nom) / (hi - nom), torch.where(y < nom, (nom - y) / (nom - lo), torch.zeros_like(y)))
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf)


def linear_c_needed(y: torch.Tensor, ref: dict) -> float:
    """The smallest of 0, 2^-6 LINEAR_C, ..., LINEAR_C under which y passes (inf if none does)."""
    for c in [0.0] + [LINEAR_C * 2.0 ** -i for i in range(6, -1, -1)]:
        if float(linear_ratios(y, ref, c).max()) <= 1:
            return c
    return math.inf


def linear_rows(M: int, K: int, gen: torch.Generator, device: str = "cpu") -> torch.Tensor:
    """bf16 [M, K] activations of the linear tests: randn rows, row 0 scaled by 1e-3, row M - 1 by 1e3 and row M // 2 zero (where
    those rows are distinct)."""
    x = torch.randn(M, K, generator=gen, device=device)
    used = set()
    for m, scale in ((0, 1e-3), (M - 1, 1e3), (M // 2, 0.0)):
        if m not in used:
            x[m] *= scale
            used.add(m)
    return x.bfloat16()


# ---- Mimi's tensor-core layers: the plan runs, and one layer against fp64 ----------------------------------------------------
def _gen_mimi_plans():
    import sys
    from pathlib import Path
    tools = str(Path(__file__).resolve().parent.parent / "tools")
    if tools not in sys.path:
        sys.path.insert(0, tools)
    import gen_mimi_plans
    return gen_mimi_plans


@functools.lru_cache(maxsize=4)
def _mimi_plan_runs(lib, sms: int, max_b: int) -> dict:
    shapes, runs, frame = _gen_mimi_plans().plan_runs(sms, max_b, lib)
    return {"shapes": shapes, "runs": runs, "frame": frame}


def mimi_plan_runs(lib, sms: int, max_b: int = 512) -> dict:
    """b200_op_mimi_plan at 1..max_b sessions on ``sms`` SMs for the default MimiConfig, compressed as tools/gen_mimi_plans.py
    writes tests/golden/mimi_plans.json: "shapes" {layer: SHAPE}, "runs" {layer: [[B_first, B_last, FIELDS]]} and "frame"
    [[B_first, B_last, FRAME]] (the field lists of that tool)."""
    return _mimi_plan_runs(lib, sms, max_b)


def mimi_plan_batches(lib, sms: int, max_b: int = 512) -> list[int]:
    """The first and last session count of every run of mimi_plan_runs (layers and frame), ascending."""
    t = mimi_plan_runs(lib, sms, max_b)
    return sorted({b for runs in [t["frame"], *t["runs"].values()] for r in runs for b in r[:2]})


# Acceptance rule of one 3xTF32 layer (mimi_tc_kernel, with or without its split-K reduction): every output within
# tc_c(chain) * 2^-24 * scale of the fp64 layer, scale = sum_k |a_k w_k| + |bias| over the products that make the output (a
# the activated input).  TC_C covers, per product, the dropped a_lo * w_lo term and the tf32 rounding of the lo parts (about
# 3 * 2^-22 together), fp32 accumulation in any order (k-blocks, splits, the split-order reduction), and fp32 expm1f in the
# ELU, for accumulation chains of up to TC_CHAIN k-blocks.  The tensor cores' fp32 accumulation is not a rounded-to-nearest
# chain: on one H100 80GB HBM3 (power limit 700 W) a layer's need grew as about 6.3 sqrt(k-blocks per split), from 9 at one
# k-block to 61 at encoder.9's 96 unsplit k-blocks (257..512 sessions), while an fp32 emulation needs at most 5 at any
# length.  Longer chains therefore get TC_C sqrt(chain / TC_CHAIN) (tc_c).  tests/test_mimi_plan_runs_cpu.py pins both,
# shows that fp32 emulations pass in several orders at every plan run of the golden table and that the kernel bugs it lists
# are rejected in every output row they touch.
TC_C = 32.0
TC_CHAIN = 8


def tc_c(chain: int) -> float:
    """The rule's constant for a layer whose k-blocks run in chains of ``chain`` (the plan's kb_per_split)."""
    return TC_C * max(1.0, (chain / TC_CHAIN) ** 0.5)
TC_CONV, TC_CONVTR, TC_LINEAR = 0, 1, 2


def tc_ref64(kind: int, x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, prev: torch.Tensor | None = None,
             stride: int = 1, dil: int = 1, elu: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """(want, scale) of one tensor-core layer in float64, on x's device, as b200_op_tc_conv1d / b200_op_tc_linear_f32 state it:
      conv:    y = conv1d(cat(prev, act(x)), w, bias, stride, dil), x [B, Cin, T], w [Cout, Cin, k], prev [B, Cin, P]
               (P = (k - 1) dil + 1 - stride; absent: zeros) -> [B, Cout, T / stride];
      convtr:  StreamingConvTranspose1d with k = 2 stride as two taps over [x[t-1], x[t]], x[-1] = prev [B, Cin, 1]:
               y[b, co, t S + r] = bias[co] + x[t] . w[:, co, r] + x[t-1] . w[:, co, S + r], w [Cin, Cout, 2 S] -> [B, Cout, T S];
      linear:  y = x . w^T, x [M, K], w [N, K] -> [M, N].
    act is ELU with ``elu`` (fp64 here), identity otherwise; the carried context ``prev`` is already activated.  scale is the
    same layer on |act|, |w| plus |bias|."""
    f64 = torch.float64
    if kind == TC_LINEAR:
        xd, wd = x.to(f64), w.to(x.device, f64)
        return xd @ wd.T, xd.abs() @ wd.abs().T
    B, Cin, T = x.shape
    a = x.to(f64)
    a = F.elu(a) if elu else a
    wd = w.to(x.device, f64)
    bd = torch.zeros(wd.shape[1] if kind == TC_CONVTR else wd.shape[0], dtype=f64, device=x.device) if bias is None \
        else bias.to(x.device, f64)
    if kind == TC_CONVTR:
        S = wd.shape[-1] // 2
        ctx = torch.zeros(B, Cin, 1, dtype=f64, device=x.device) if prev is None else prev.to(x.device, f64)
        ext = torch.cat([ctx, a], dim=-1)
        # taps (x[t-1], x[t]) of phase r: [S, Cout, Cin, 2] -> [S Cout, Cin, 2]
        taps = torch.stack([wd[:, :, S:], wd[:, :, :S]], dim=-1).permute(2, 1, 0, 3).reshape(S * wd.shape[1], Cin, 2)

        def run(e, k, b):
            y = F.conv1d(e, k, b.repeat(S))                                  # [B, S Cout, T]: channel r Cout + co
            return y.view(B, S, -1, T).permute(0, 2, 3, 1).reshape(B, -1, T * S)
        return run(ext, taps, bd), run(ext.abs(), taps.abs(), bd.abs())
    k = wd.shape[-1]
    P = (k - 1) * dil + 1 - stride
    ctx = torch.zeros(B, Cin, P, dtype=f64, device=x.device) if prev is None else prev.to(x.device, f64)
    ext = torch.cat([ctx, a], dim=-1)
    return (F.conv1d(ext, wd, bd, stride=stride, dilation=dil),
            F.conv1d(ext.abs(), wd.abs(), bd.abs(), stride=stride, dilation=dil))


def tc_ratios(got: torch.Tensor, want: torch.Tensor, scale: torch.Tensor, c: float = TC_C) -> torch.Tensor:
    """|got - want| / (c 2^-24 scale) per output (<= 1 passes).  Where scale is 0 only an exact 0 passes; a NaN never does."""
    want = want.double()
    got = got.detach().to(want.device, torch.float64).reshape(want.shape)
    tol = c * 2.0 ** -24 * scale.double()
    err = (got - want).abs()
    r = torch.where(tol > 0, err / tol, torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    return torch.nan_to_num(r, nan=math.inf, posinf=math.inf)


def tc_rows(r: torch.Tensor, kind: int, stride: int = 1) -> torch.Tensor:
    """Per-output values of one layer [B, Cout, T'] (or [M, N]) regrouped by GEMM row: [B, T, outputs of the row] (a
    transposed conv's GEMM row t holds its output steps t S .. t S + S - 1); a linear's [M, N] becomes [M, 1, N]."""
    if kind == TC_LINEAR:
        return r[:, None]
    B, Co, Tr = r.shape
    S = stride if kind == TC_CONVTR else 1
    return r.view(B, Co, Tr // S, S).permute(0, 2, 1, 3).reshape(B, Tr // S, Co * S)


def mimi_tc_layers(cfg) -> dict[str, dict]:
    """The tensor-core layers of b200_op_mimi_plan by name ("encoder.<i>" / "decoder.<i>": position i in the handle's list of
    SEANet convolutions, a resnet block giving two; "transformer.<linear>"), each with what b200_op_tc_conv1d takes: kind
    (TC_CONV / TC_CONVTR; the transformer linears as 1-tap convs), cin, cout, k, stride, dil and elu (ELU on the input).
    Restates the module order of synth.seanet_layout; the first encoder and the last decoder conv (one channel) are not
    tensor-core layers."""
    from moshi_b200.synth import seanet_layout
    out = {}
    for side, layout in zip(("encoder", "decoder"), seanet_layout(cfg)):
        convs = []
        for kind, _, cin, cout, k, stride, dil in layout:
            if kind == "res":
                hid = cin // cfg.compress
                convs += [(TC_CONV, cin, hid, k, 1, dil), (TC_CONV, hid, cout, 1, 1, 1)]
            else:
                convs.append((TC_CONVTR if kind == "convtr" else TC_CONV, cin, cout, k, stride, dil))
        for i, (kind, cin, cout, k, stride, dil) in enumerate(convs):
            if cin == 1 or cout == 1:
                continue
            out[f"{side}.{i}"] = dict(kind=kind, cin=cin, cout=cout, k=k, stride=stride, dil=dil, elu=i > 0)
    d, ff = cfg.tr_d_model, cfg.tr_dim_feedforward
    for name, cin, cout in (("in_proj", d, 3 * d), ("out_proj", d, d), ("linear1", d, ff), ("linear2", ff, d)):
        out[f"transformer.{name}"] = dict(kind=TC_CONV, cin=cin, cout=cout, k=1, stride=1, dil=1, elu=False)
    return out


def tc_op_shape(layer: dict, T_rows: int) -> list[int]:
    """What b200_op_tc_conv1d plans for ``layer`` (mimi_tc_layers) at T_rows GEMM rows per session, in the order of
    gen_mimi_plans.SHAPE without the kind: Cin, N, taps, dilation, stride, NT, feature tiles, k-blocks, T.  Its input has
    T_rows * stride steps (T_rows for a transposed conv)."""
    tr = layer["kind"] == TC_CONVTR
    N = layer["stride"] * layer["cout"] if tr else layer["cout"]
    taps = 2 if tr else layer["k"]
    NT = min(N, 128)
    return [layer["cin"], N, taps, 1 if tr else layer["dil"], 1 if tr else layer["stride"], NT, -(-N // NT),
            taps * (layer["cin"] // 32), T_rows]
