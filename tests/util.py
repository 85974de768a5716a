"""Shared helpers for the GPU parity tests."""
from __future__ import annotations

import ctypes as C
import functools
import math

import torch


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
    """Round to bf16 and back (a cast point of the bf16 model)."""
    return x.to(torch.bfloat16).to(x.dtype)


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
                    mutant: dict | None = None) -> dict:
    """One depformer frame (lm.py:450-493 and 809-850 with transformer.py's weights-per-step layers, as oracle/lm.py
    forward_depformer / depformer_step state it) in float64, teacher-forced: sub-step k's previous token is ``text_token`` [B]
    for k = 0 and ``audio_tokens[k - 1]`` ([dep_q, B], the tokens the model under test sampled) after.  Values are rounded to
    bf16 at the cast points of the bf16 model (csrc/dep_fused.cu):
      x = bf16(bf16(din_k) + emb_k(prev));  xn = bf16(rmsnorm(x));  q, k, v = bf16(in_proj(xn));
      out = bf16(softmax(q . k_j / 8) . v_j over the keys j = 0..k);  x = bf16(x + bf16(out_proj(out)));
      h = bf16(bf16(silu(bf16 g)) * bf16 u);  x = bf16(x + bf16(linear_out(h)));  logits = linears[k](x).
    Runs on transformer_out's device.  Weights are converted to float64 one (sub-step, layer) at a time, never all at once.

    Returns the checkpoints before their final bf16 rounding, as float64: "din" [B, dep_q, dd] (depformer_in[k] of
    transformer_out), "k" / "v" per layer [B, H, dep_q, 64] (what the layer's per-frame cache holds after the frame) and
    "logits" [dep_q, B, card].

    ``mutant`` (for the tests of the acceptance rule) replaces parts of the computation:
      "weight": f(name, k, layer, fetch) -> the raw tensor to use, where fetch(name, k, layer) gives the right one (names:
                din, emb, in, out, lin_in, lin_out, n1, n2, head);
      "keys":   f(k, layer) -> (lo, hi): the keys the sub-step attends over (default (0, k + 1));
      "prev":   f(k, tokens) -> the previous tokens of sub-step k, tokens = [text_token, audio_tokens[0], ...];
      "residual": f(k, layer, "attn" | "ffn") -> False to drop that residual."""
    mutant = mutant or {}
    dev, f64 = transformer_out.device, torch.float64
    B = transformer_out.shape[0]
    dd, H, L, Q = cfg.depformer_dim, cfg.depformer_num_heads, cfg.depformer_num_layers, cfg.dep_q
    D = dd // H

    def fetch(name, k, layer=None):
        return _dep_tensor(sd, name, k, layer)

    def W(name, k, layer=None):
        t = mutant["weight"](name, k, layer, fetch) if "weight" in mutant else fetch(name, k, layer)
        if name == "emb":
            return t                                    # only the rows of the previous tokens are gathered and converted
        t = t.to(dev, f64)
        return t.reshape(-1) if name in ("n1", "n2") else t

    def rmsnorm(x, alpha):
        return _bf(x * alpha / torch.sqrt(1e-8 + x.pow(2).mean(-1, keepdim=True)))

    tout = transformer_out.to(f64)
    tokens = [text_token.to(dev)] + [audio_tokens[k].to(dev) for k in range(Q - 1)]
    din = torch.stack([tout @ W("din", k).T for k in range(Q)], dim=1)
    kc = [torch.zeros(B, H, Q, D, dtype=f64, device=dev) for _ in range(L)]
    vc = [torch.zeros(B, H, Q, D, dtype=f64, device=dev) for _ in range(L)]
    logits = []
    for k in range(Q):
        prev = mutant["prev"](k, tokens) if "prev" in mutant else tokens[k]
        table = W("emb", k)
        e = table.to(dev)[prev.clamp(min=0)].to(f64) * (prev >= 0)[:, None]          # token -1 -> zero row (lm_utils.py:103-121)
        x = _bf(_bf(din[:, k]) + e)
        for layer in range(L):
            xn = rmsnorm(x, W("n1", k, layer))
            qkv = (xn @ W("in", k, layer).T).view(B, 3, H, D)
            kc[layer][:, :, k], vc[layer][:, :, k] = qkv[:, 1], qkv[:, 2]
            lo, hi = mutant["keys"](k, layer) if "keys" in mutant else (0, k + 1)
            s = torch.einsum("bhd,bhnd->bhn", _bf(qkv[:, 0]), _bf(kc[layer][:, :, lo:hi])) * 0.125
            o = _bf(torch.einsum("bhn,bhnd->bhd", torch.softmax(s, dim=-1), _bf(vc[layer][:, :, lo:hi]))).reshape(B, dd)
            upd = _bf(o @ W("out", k, layer).T)
            x = _bf(x + upd) if mutant.get("residual", lambda *a: True)(k, layer, "attn") else upd
            xn = rmsnorm(x, W("n2", k, layer))
            gu = xn @ W("lin_in", k, layer).T
            F_ = gu.shape[1] // 2
            g, u = _bf(gu[:, :F_]), _bf(gu[:, F_:])
            h = _bf(_bf(g * torch.sigmoid(g)) * u)
            upd = _bf(h @ W("lin_out", k, layer).T)
            x = _bf(x + upd) if mutant.get("residual", lambda *a: True)(k, layer, "ffn") else upd
        logits.append(x @ W("head", k).T)                                             # depformer_norms is Identity (lm.py:197-198)
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
DEP_C_DIN = 2.0 ** -10
DEP_C_KV = (2.0 ** -8, 0.025, 0.04, 0.05, 0.0625, 0.094)
DEP_C_LOGITS = 0.08


def dep_c_kv(layer: int) -> float:
    return DEP_C_KV[min(layer, len(DEP_C_KV) - 1)]


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


def dep_c(kind: str, layer: int | None) -> float:
    return DEP_C_DIN if kind == "din" else DEP_C_LOGITS if kind == "logits" else dep_c_kv(layer)


def dep_row_ratios(got: torch.Tensor, want: torch.Tensor, kind: str, layer: int | None) -> torch.Tensor:
    """Worst err_ratios of each batch row of one checkpoint under its constant: [B] (<= 1 passes)."""
    r = err_ratios(got, want, dep_c(kind, layer))
    return r.reshape(r.shape[0], -1).amax(dim=1)
