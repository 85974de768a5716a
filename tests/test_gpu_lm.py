"""GPU: Moshi LM decode step (LMGen.step) against the CPU oracle and the reference-recorded fixtures."""
import pytest
import torch
from safetensors.torch import load_file

from moshi_b200.config import LMConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict
from oracle import scenarios
from oracle.lm import LMOracle, LMSpec, sample_token

pytestmark = pytest.mark.gpu

# bf16 logits: half an ulp at |x|~4 is 0.016; accumulation order moves a result across a rounding
# boundary now and then, and the difference propagates through the layers.
LOGIT_ATOL = 0.08


@pytest.fixture(scope="module")
def tiny():
    cfg = tiny_lm_config()
    return cfg, synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)


@pytest.fixture(scope="module")
def lm(tiny):
    from moshi_b200.models import LMModel
    cfg, sd = tiny
    return LMModel(cfg, sd, device="cuda")


def test_attributes_match_reference(lm):
    assert (lm.n_q, lm.dep_q, lm.card, lm.num_codebooks) == (16, 8, 64, 17)
    assert lm.delays == [0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1]
    assert lm.dtype == torch.bfloat16 and lm.device.type == "cuda"
    assert (lm.zero_token_id, lm.ungenerated_token_id, lm.initial_token_id) == (-1, -2, 64)


def _run(lm, tiny, sampling, use_graph, golden, quantize=False, record=None):
    """Teacher-synchronised comparison: the oracle is stepped on the GPU's own token stream, so a
    single near-tie flip does not make every later step incomparable."""
    from moshi_b200.models import LMGen
    cfg, sd = tiny
    B, steps = scenarios.LM_B, scenarios.LM_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps)
    gen = LMGen(lm, use_sampling=sampling, temp=0.8, temp_text=0.7)
    gen.use_graph = use_graph
    # ties among bf16 logits are ranked by token id on the GPU; torch.topk's order is unspecified
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=sampling, tie_break="index", quantize=quantize)
    orc.streaming(B)
    diverged = torch.zeros(B, dtype=torch.bool)    # rows whose token history left the reference trajectory
    torch.manual_seed(scenarios.LM_NOISE_SEED)
    tok_match = tok_total = 0
    gold_match = gold_total = 0
    samp_match = samp_total = 0      # sampler exactness: oracle sampler applied to the GPU's own logits
    worst = 0.0
    report = []
    with gen.streaming(B):
        for i in range(steps):
            scenarios.lm_mask_events(gen, i, B)
            scenarios.lm_mask_events(orc, i, B)
            nt, na = scenarios.lm_noise(cfg, B) if sampling else (None, None)
            dbg = {}
            want = orc.step(codes[i], nt, na, debug=dbg)
            noise = gen.pack_noise(nt, na) if sampling else None
            got = gen.step(codes[i].cuda(), noise=noise)
            live = orc.exec_mask
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            tl_o = dbg["text_logits"].float()[:, 0, 0]
            d = (tl - tl_o)[live].abs().max().item()
            worst = max(worst, d)
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu()
            dl_o = torch.stack([x.float()[:, 0, 0] for x in dbg["dep_logits"]])
            # depformer sub-step k>0 depends on the previously sampled token: compare where tokens agree
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            if record is not None:      # what the GPU sampled this step and the logits it sampled from
                record.append((orc.exec_mask.clone(), torch.cat([tt[:, None], at.t()], 1), [tl] + [dl[k] for k in range(cfg.dep_q)],
                               torch.cat([dbg["text_token"][:, None], dbg["audio_tokens"]], 1)))
            if sampling:
                want_t = sample_token(tl, True, 0.7, 25, nt, "index")
                samp_match += int((want_t == tt)[live].sum())
                samp_total += int(live.sum())
                for k in range(cfg.dep_q):
                    want_a = sample_token(dl[k], True, 0.8, 250, na[k], "index")
                    samp_match += int((want_a == at[k])[live].sum())
                    samp_total += int(live.sum())
            same_text = (tt == dbg["text_token"]) & live
            if same_text.any():
                worst = max(worst, (dl[0] - dl_o[0])[same_text].abs().max().item())
            report.append(f"step {i}: text_logits max diff {d:.3e}; text tokens equal {int(same_text.sum())}/{int(live.sum())}")
            assert (want is None) == (got is None), i
            if i == 20:
                diverged[1] = False           # scenarios.lm_mask_events: row 1 restarts from scratch
            diverged |= live & ((tt != dbg["text_token"]) | (at.t() != dbg["audio_tokens"]).any(dim=1))
            if got is not None:
                ok = (got.cpu() == want)[live]
                tok_match += int(ok.sum())
                tok_total += ok.numel()
                if golden is not None:
                    # the fixture is a free-running reference run: only rows that are still on the
                    # reference's token trajectory can be compared with it, and those must be equal
                    g = golden["tokens"][i]
                    sel = live & ~diverged
                    okg = (got.cpu() == g)[sel]
                    gold_match += int(okg.sum())
                    gold_total += okg.numel()
            # keep the oracle on the GPU's trajectory: overwrite what it just stored in its token ring
            if not torch.equal(tt[live], dbg["text_token"][live]) or not torch.equal(at.t()[live], dbg["audio_tokens"][live]):
                pos = (orc.offsets % orc.cache.shape[2])
                for b in range(B):
                    if live[b]:
                        orc.cache[b, 0, pos[b]] = tt[b]
                        orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print("\n".join(report[:6]))
    print(f"sampling={sampling} graph={use_graph}: tokens equal to oracle {tok_match}/{tok_total}, "
          f"to reference fixture {gold_match}/{gold_total}, worst logit diff {worst:.3e}, "
          f"sampler on the GPU's own logits {samp_match}/{samp_total}")
    return tok_match, tok_total, gold_match, gold_total, worst, samp_match, samp_total


def _reference_trajectory(cfg, rec, gold_tokens, restarts):
    """The GPU against a free-running reference run (the fixture): a row is on the reference's trajectory while every token it
    sampled so far equals the reference's.  On such a row a sampled token that differs from the reference's takes the row off
    the trajectory, and is excused in two cases only: the GPU also differs from the oracle there (a GPU-vs-oracle flip, bounded
    by the agreement rate the caller asserts), or the GPU's own logits rank its token and the reference's within
    ``2 * LOGIT_ATOL`` (a near-tie that the CPU's bf16 matmul path, which differs between CPUs, decides either way).
    ``rec`` holds per step (live rows, tokens [B, 1 + dep_q] as the GPU sampled them, the GPU's logits per codebook [B, card],
    the oracle's tokens); the fixture holds the delayed outputs, so the token sampled at step i for codebook k is output
    ``i + max_delay - delay_k``; a row whose token is missing from the fixture leaves the trajectory.  ``restarts``: {step: rows that restart from scratch}.  Returns (compared, unexcused)."""
    n_tok = 1 + cfg.dep_q
    max_delay = max(cfg.delays[:n_tok])
    steps = len(rec)
    B = rec[0][0].shape[0]
    off = torch.zeros(B, dtype=torch.bool)
    compared = unexcused = 0
    for i, (live, toks, logits, orc_toks) in enumerate(rec):
        if i + max_delay >= steps:      # the fixture ends before this step's tokens are all output: its history is unknown
            break
        for b in restarts.get(i, ()):
            off[b] = False
        for k in range(n_tok):
            j = i + max_delay - cfg.delays[k]
            ref = gold_tokens[j][:, k, 0]
            sel = live & rec[j][0] & ~off
            for b in sel.nonzero().flatten().tolist():
                if not 0 <= int(ref[b]) < logits[k].shape[1]:
                    # not in the fixture: the first max_delay outputs are empty by construction; any other missing output
                    # (the step of a reset returns none) hides a token the row went on with, so its history is unknown
                    if j >= max_delay:
                        off[b] = True
                    continue
                compared += 1
                g, r = int(toks[b, k]), int(ref[b])
                if g != r:
                    gap = float(logits[k][b, g] - logits[k][b, r])
                    if g == int(orc_toks[b, k]) and gap >= 2 * LOGIT_ATOL:
                        unexcused += 1
                        print(f"unexcused: step {i} codebook {k} row {b}: GPU {g}, reference {r}, GPU logit gap {gap:.3f}")
                    off[b] = True
    return compared, unexcused


@pytest.mark.parametrize("use_graph", [False, True])
def test_greedy_steps_match_oracle_and_reference(lm, tiny, golden_dir, use_graph):
    gold = load_file(golden_dir / "lm_tiny_greedy.safetensors")
    rec = []
    m, t, _, _, worst, _, _ = _run(lm, tiny, False, use_graph, gold, record=rec)
    assert worst < LOGIT_ATOL
    assert m / t > 0.97          # greedy flips only on bf16 logit near-ties
    # rows still on the reference's own trajectory reproduce the fixture, up to flips on provable bf16 near-ties
    # (scenarios.lm_mask_events: row 1 restarts from scratch at step 20)
    compared, unexcused = _reference_trajectory(tiny[0], rec, gold["tokens"], {20: (1,)})
    print(f"against the reference fixture: {compared} tokens compared on its trajectory, {unexcused} unexcused")
    assert compared > 0 and unexcused == 0


@pytest.mark.parametrize("use_graph", [False, True])
def test_sampled_steps_match_oracle_and_reference(lm, tiny, golden_dir, use_graph):
    gold = load_file(golden_dir / "lm_tiny_sampled.safetensors")
    m, t, gm, gt, worst, sm, st = _run(lm, tiny, True, use_graph, gold)
    assert worst < LOGIT_ATOL
    # Sampled ids are bit-exact *given the logits*: the reference sampler (ties ranked by token id) run on the
    # GPU's own bf16 logits with the same Exp(1) noise reproduces every GPU token.  Against the oracle's own
    # logits the ids only agree where the bf16 rounding noise (<= LOGIT_ATOL) does not reorder candidates: the
    # noise is indexed by rank (sampling.py:62-64), so on this random-weight model (near-uniform distributions,
    # 64 candidates all inside the top-k) a one-ulp swap re-deals the noise.  That rate is reported, not gated.
    assert st > 0 and sm >= st - 1
    assert m / t > 0.5
    # torch.topk's order among tied probabilities is unspecified, so the free-running sampled fixture is
    # only reported (gm/gt printed by _run); the exact claims are the greedy fixture and the oracle above


def test_step_outside_streaming_raises(lm):
    from moshi_b200.models import LMGen
    gen = LMGen(lm)
    with pytest.raises(RuntimeError):
        gen.step(torch.zeros(1, 8, 1, dtype=torch.long, device="cuda"))
    with gen.streaming(2):
        with pytest.raises(AssertionError):
            gen.step(torch.zeros(1, 8, 1, dtype=torch.long, device="cuda"))
        with pytest.raises(AssertionError):
            gen.step(torch.zeros(2, 3, 1, dtype=torch.long, device="cuda"))


@torch.no_grad()
def test_shortened_kv_ring_is_the_reference_ring_until_it_is_full(lm, tiny):
    """`kv_capacity` (b200_lm_set_kv_capacity; SURVEY 8f item 3, rings sized to live fill): a ring of 8 slots gives the same
    logits and tokens as the model's own 12-slot ring for a session's first 8 frames (nothing is evicted before position
    `context`), and the frame that would overwrite a live key raises error flag 4 instead of silently forgetting."""
    from moshi_b200.models import LMGen
    cfg, _ = tiny
    B, cap = 4, 8
    assert cap < cfg.context
    g = torch.Generator().manual_seed(99)
    codes = torch.randint(0, cfg.card, (cap + 1, B, 8, 1), generator=g).cuda()
    outs = {}
    for name, kv_capacity in (("full", None), ("short", cap)):
        gen = LMGen(lm, use_sampling=False, check=False)
        gen.kv_capacity = kv_capacity
        rec = []
        with gen.streaming(B):
            for i in range(cap):
                gen.step(codes[i])
                rec.append((gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).cpu(),
                            gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()))
            assert gen.error_flags() == 0
            if kv_capacity is not None:
                gen.step(codes[cap])                       # position 8 of an 8-slot ring
                assert gen.error_flags() == 4
                assert gen.error_flags() == 0              # reading clears
        outs[name] = rec
    same = total = 0
    for (tl_f, at_f), (tl_s, at_s) in zip(outs["full"], outs["short"]):
        # the same keys in the same order: equal up to the fp32 summation order of the attention's key groups
        torch.testing.assert_close(tl_s.float(), tl_f.float(), rtol=0, atol=LOGIT_ATOL)
        same += int((at_f == at_s).sum())
        total += at_f.numel()
    assert same / total >= 0.97, (same, total)


@torch.no_grad()
def test_rows_independent_graph_invariant_and_host_path():
    """Mid-size member of the 7B family at a serving batch, full 3000-slot ring machinery:
    (1) graph replay == eager launches bit for bit, (2) a session's tokens do not depend on its slot or its neighbours
    (the batch with its rows reversed gives the reversed tokens; a *different batch size* may run other kernels — the GEMV
    path below five sessions, other split points — so "alone" is only equal up to summation order and is checked on the
    7B model's logits below), (3) the host-buffer entry point returns the same tokens, (4) masked rows do not advance."""
    from moshi_b200.models import LMGen, LMModel
    cfg = LMConfig(dim=1024, num_heads=8, num_layers=4, context=3000, text_card=32000, card=2048,
                   depformer_dim=512, depformer_num_heads=8, depformer_dim_feedforward=2112, depformer_num_layers=2)
    lm = LMModel(cfg, synth_lm_state_dict(cfg, seed=5, device="cuda"), device="cuda")
    B, steps = 24, 6
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, cfg.card, (steps, B, 8, 1), generator=g).cuda()
    noise = torch.empty(steps, B, 25 + 8 * 250).exponential_(1, generator=g).cuda()

    def run(batch_rows, use_graph, host=False, fill=0, mask_row=None):
        gen = LMGen(lm)
        gen.use_graph = use_graph
        outs = []
        with gen.streaming(len(batch_rows)):
            if fill:
                gen.assume_fill(fill)
            for i in range(steps):
                if mask_row is not None:
                    m = torch.ones(len(batch_rows), dtype=torch.bool)
                    m[mask_row] = i not in (2, 3)
                    gen.set_exec_mask(m)
                c, n = codes[i][batch_rows], noise[i][batch_rows].contiguous()
                if host:
                    o = torch.empty(len(batch_rows), 9, dtype=torch.int64)
                    ready = gen.step_host(c[:, :, 0].cpu().contiguous(), n.cpu(), o)
                    outs.append(o if ready else None)
                else:
                    o = gen.step(c, noise=n)
                    outs.append(None if o is None else o[:, :, 0].cpu())
        return outs

    rows = list(range(B))
    eager = run(rows, False)
    graph = run(rows, True)
    host = run(rows, True, host=True)
    flipped = run(rows[::-1], True)
    assert eager[0] is None and eager[1] is not None      # max_delay = 1: offset_cpu <= max_delay -> None (lm.py:774-776)
    for i in range(1, steps):
        assert torch.equal(eager[i], graph[i]), i
        assert torch.equal(eager[i], host[i]), i
        assert torch.equal(eager[i], flipped[i].flip(0)), i
        assert (eager[i] >= 0).all() and (eager[i][:, 1:] < cfg.card).all() and (eager[i][:, 0] < cfg.text_card).all()
    # ring wrap-around: positions near the 3000-slot capacity
    wrapped = run(rows, True, fill=2998)
    assert all(o is not None for o in wrapped)
    # assume_fill leaves the token ring "ungenerated" (-2): the first output re-aligns the previous step's slot
    assert all((o >= 0).all() for o in wrapped[1:])
    masked = run(rows, True, mask_row=3)
    for i in (2, 3):
        assert (masked[i][3] == -2).all()
        assert torch.equal(masked[i][[0, 1, 2] + list(range(4, B))], eager[i][[0, 1, 2] + list(range(4, B))])


def test_depformer_replace_tokens(lm, tiny):
    """``LMGen.step(codes, depformer_replace_tokens=...)`` (lm.py:751-755, the TTS caller): the given audio tokens enter the
    ring instead of the depformer's, the text token is still sampled; frames with and without replacement alternate
    (two captured graphs), and the stream stays on the oracle's trajectory."""
    from moshi_b200.models import LMGen
    cfg, sd = tiny
    B, steps = 3, 10
    codes = scenarios.lm_input_codes(cfg, B, steps)
    g = torch.Generator().manual_seed(3)
    forced = torch.randint(0, cfg.card, (steps, B, cfg.dep_q, 1), generator=g)
    gen = LMGen(lm, use_sampling=False)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, tie_break="index")
    orc.streaming(B)
    agree = total = 0
    with gen.streaming(B):
        for i in range(steps):
            rep = forced[i] if i % 3 != 2 else None
            dbg = {}
            want = orc.step(codes[i], None, None, debug=dbg, depformer_replace_tokens=rep)
            got = gen.step(codes[i].cuda(), depformer_replace_tokens=None if rep is None else rep.cuda())
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            if rep is not None:
                assert torch.equal(at.t(), rep[:, :, 0])            # forced tokens are what the ring receives
            assert (want is None) == (got is None)
            if got is not None:
                agree += int((got.cpu() == want).sum())
                total += want.numel()
            # keep the oracle on the GPU's trajectory (greedy near-ties)
            pos = (orc.offsets % orc.cache.shape[2])
            for b in range(B):
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print(f"replace tokens: {agree}/{total} output tokens equal to the oracle")
    assert agree / total > 0.95


def test_full_size_7b_properties():
    """BASELINE's own configuration (configs/moshi_7b_202409.json, random block-tiled weights) is too large for the CPU
    oracle, so the full-size step is checked through size-independent properties: graph replay == eager launches; a
    session's tokens do not depend on its slot or on its neighbours (no cross-row op anywhere, SURVEY 8e: the batch with
    its rows permuted gives the permuted tokens, bit for bit); alone in a batch of one the same session gives the same
    logits up to the fp32 summation order of the split-KV / split-K schedules, which are chosen per batch size; paused
    rows do not move; outputs in range; the ring wraps at slot 3000."""
    from moshi_b200.config import MOSHI_7B
    from moshi_b200.models import LMGen, loaders
    lm7 = loaders.get_moshi_lm(None, MOSHI_7B.to_reference_kwargs(), device="cuda", synth_device="cuda")
    cfg = MOSHI_7B
    B, steps = 5, 5
    g = torch.Generator().manual_seed(11)
    codes = torch.randint(0, cfg.card, (steps, B, 8, 1), generator=g).cuda()
    noise = torch.empty(steps, B, 25 + 8 * 250).exponential_(1, generator=g).cuda()

    def run(rows, use_graph, fill=2997, paused=None, logits=None):
        gen = LMGen(lm7)
        gen.use_graph = use_graph
        outs = []
        with gen.streaming(len(rows)):
            gen.assume_fill(fill)                      # steps cross the ring's wrap at 3000
            for i in range(steps):
                if paused is not None:
                    m = torch.ones(len(rows), dtype=torch.bool)
                    m[paused] = i != 2
                    gen.set_exec_mask(m)
                o = gen.step(codes[i][rows], noise=noise[i][rows].contiguous())
                outs.append(o[:, :, 0].cpu())
                if logits is not None and i == 0:
                    logits.append(gen.read_buffer("text_logits", torch.bfloat16, (len(rows), cfg.text_card)).float().cpu())
        return outs

    rows = list(range(B))
    perm = [4, 2, 0, 3, 1]
    la, ls = [], []
    eager, graph, shuffled = run(rows, False, logits=la), run(rows, True), run(perm, True)
    run([3], True, logits=ls)
    paused = run(rows, True, paused=1)
    d = (la[0][3] - ls[0][0]).abs().max().item()
    print(f"7B: text logits of session 3 in a batch of {B} vs alone: max |d| = {d:.3e}")
    # alone, the linears take the GEMV path (fp32 FMA chains) instead of the tensor-core GEMM: another summation order in every
    # one of the 32 layers' four linears; bf16 rounding noise (2^-9 per cast) random-walks to ~0.2 on logits of |x| ~ 4
    assert d < 0.35
    for i in range(1, steps):
        assert torch.equal(eager[i], graph[i]), i
        assert torch.equal(eager[i][perm], shuffled[i]), i
        assert (eager[i] >= 0).all() and (eager[i][:, 1:] < cfg.card).all() and (eager[i][:, 0] < cfg.text_card).all()
    assert (paused[2][1] == -2).all()
    keep = [0, 2, 3, 4]
    for i in range(1, steps):
        assert torch.equal(paused[i][keep], eager[i][keep]), i
    del lm7
    torch.cuda.empty_cache()


@torch.no_grad()
def test_streaming_state_snapshot_roundtrip(lm, tiny):
    """LMGen.get_streaming_state / set_streaming_state: the continuation from a snapshot is reproduced exactly."""
    from moshi_b200.models import LMGen
    cfg, _ = tiny
    B = 2
    g = torch.Generator().manual_seed(3)
    codes = torch.randint(0, cfg.card, (8, B, 8, 1), generator=g).cuda()
    gen = LMGen(lm, use_sampling=False)
    with gen.streaming(B):
        for i in range(4):
            gen.step(codes[i])
        snap = gen.get_streaming_state()
        first = [gen.step(codes[i]).cpu() for i in range(4, 8)]
        gen.set_streaming_state(snap)
        second = [gen.step(codes[i]).cpu() for i in range(4, 8)]
    for a, b in zip(first, second):
        assert torch.equal(a, b)


@torch.no_grad()
@pytest.mark.parametrize("B", [17, 130])
def test_fused_depformer_equals_launch_chain(B):
    """The persistent depformer kernel against the per-kernel launch chain on a mid-size member of the 7B family, at batch
    sizes that exercise odd paddings (Mpad 32 / 144, two launches above 128 sessions) and the cluster
    split-K GEMMs: same text logits, same depformer logits within bf16 accumulation-order noise, near-identical greedy ids."""
    from moshi_b200 import _lib
    from moshi_b200.models import LMGen, LMModel
    cfg = LMConfig(dim=1024, num_heads=8, num_layers=2, context=64, text_card=4000, card=2048,
                   depformer_dim=1024, depformer_num_heads=16, depformer_dim_feedforward=4224, depformer_num_layers=3)
    sd = synth_lm_state_dict(cfg, seed=11, device="cuda")
    g = torch.Generator().manual_seed(B)
    codes = torch.randint(0, cfg.card, (4, B, 8, 1), generator=g).cuda()

    def run(mode: int):
        lm = LMModel(cfg, sd, device="cuda")
        _lib.check(_lib.lib().b200_lm_set_depformer(lm._h, mode))
        gen = LMGen(lm, use_sampling=False)
        outs = []
        with gen.streaming(B):
            for i in range(4):
                gen.step(codes[i])
                outs.append((gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu(),
                             gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu(),
                             gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()))
        del gen, lm
        return outs

    chain, fused = run(_lib.B200_DEPFORMER_CHAIN), run(_lib.B200_DEPFORMER_AUTO)
    same = total = 0
    on_track = torch.ones(B, dtype=torch.bool)             # rows whose sampled history is still identical in both runs
    for (tl_c, dl_c, at_c), (tl_f, dl_f, at_f) in zip(chain, fused):
        assert on_track.any()
        assert torch.equal(tl_c[on_track], tl_f[on_track])  # the temporal path is the same code in both runs
        # sub-step 0 sees identical inputs; later sub-steps only where the previously sampled ids agree
        torch.testing.assert_close(dl_f[0][on_track], dl_c[0][on_track], rtol=0, atol=LOGIT_ATOL)
        eq = (at_c == at_f)[:, on_track]
        same += int(eq.sum())
        total += eq.numel()
        on_track &= (at_c == at_f).all(dim=0)
    print(f"fused vs chain, B={B}: greedy ids equal {same}/{total} on rows with identical history")
    assert same / total > 0.9


@pytest.mark.parametrize("B", [1, 2])
def test_one_and_two_sessions_take_the_gemv_path(lm, tiny, B):
    """Below three sessions every linear runs as gemv_kernel (plain loads, RMSNorm folded into the activation staging) and
    the depformer as a launch chain: same oracle, same tolerance, teacher-synchronised greedy steps across the ring wrap."""
    from moshi_b200.models import LMGen
    cfg, sd = tiny
    steps = 16
    codes = scenarios.lm_input_codes(cfg, 3, steps)[:, :B]
    gen = LMGen(lm, use_sampling=False)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, tie_break="index")
    orc.streaming(B)
    worst = 0.0
    agree = total = 0
    with gen.streaming(B):
        for i in range(steps):
            dbg = {}
            orc.step(codes[i], None, None, debug=dbg)
            gen.step(codes[i].cuda())
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu()
            tt = gen.read_buffer("text_token", torch.int64, (B,)).cpu()
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
            worst = max(worst, (tl - dbg["text_logits"].float()[:, 0, 0]).abs().max().item())
            same_text = tt == dbg["text_token"]
            if same_text.any():
                worst = max(worst, (dl[0] - dbg["dep_logits"][0].float()[:, 0, 0])[same_text].abs().max().item())
            agree += int(same_text.sum()) + int((at.t() == dbg["audio_tokens"]).sum())
            total += B * (1 + cfg.dep_q)
            pos = (orc.offsets % orc.cache.shape[2])
            for b in range(B):
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    print(f"B={B} (GEMV path): worst logit diff {worst:.3e}, greedy tokens equal {agree}/{total}")
    assert worst < LOGIT_ATOL
    assert agree / total > 0.95


class _OracleAsDevice:
    """Stand-in with LMGen's surface used by _peaked_sampling_run, backed by a second oracle: lets the comparison logic itself be
    checked on the CPU (tests/test_sampling_gate_cpu.py)."""

    def __init__(self, sd, cfg, B):
        self.cfg, self.B = cfg, B
        self.orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=True, tie_break="index")
        self.orc.streaming(B)
        self.dbg = {}

    def set_exec_mask(self, m):
        self.orc.set_exec_mask(m)

    def reset_streaming(self, m=None):
        self.orc.reset_streaming(m)

    def step(self, codes, nt, na):
        self.dbg = {}
        return self.orc.step(codes, nt, na, debug=self.dbg)

    def outputs(self):
        d = self.dbg
        return (d["text_logits"].float()[:, 0, 0], torch.stack([x.float()[:, 0, 0] for x in d["dep_logits"]]), d["text_token"],
                d["audio_tokens"].t().contiguous())


def _peaked_sampling_run(dev, sd, cfg, gold):
    """Drives `dev` (the GPU LMGen wrapped below, or _OracleAsDevice) and a teacher-synchronised oracle through the peaked
    sampling scenario; returns the counters the test gates on."""
    from tests.util import sample_is_stable
    B, steps = scenarios.LM_B, scenarios.LM_STEPS
    codes = scenarios.lm_input_codes(cfg, B, steps)
    orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=True, tie_break="index")
    orc.streaming(B)
    torch.manual_seed(scenarios.LM_NOISE_SEED)
    on_ref = torch.ones(B, dtype=torch.bool)       # rows whose sampled history still equals the reference's
    c = dict(decisions=0, stable=0, equal=0, unexcused=0, ref_decisions=0, ref_equal=0, ref_unexcused=0, worst=0.0)
    for i in range(steps):
        scenarios.lm_mask_events(dev, i, B)
        scenarios.lm_mask_events(orc, i, B)
        nt, na = scenarios.lm_noise(cfg, B)
        dbg = {}
        want = orc.step(codes[i], nt, na, debug=dbg)
        got = dev.step(codes[i], nt, na)
        assert (want is None) == (got is None), i
        live = orc.exec_mask.clone()
        tl, dl, tt, at = dev.outputs()
        if i == 20:
            on_ref[1] = True                  # scenarios.lm_mask_events: row 1 restarts from scratch (in the reference run too)
        # sampler by sampler.  `same`: this row's inputs to the sampler are identical on the device and in the oracle, so the
        # oracle's logits are the right yardstick; `ref_same`: they also equal the reference run's (whose logits the oracle
        # reproduces bit for bit), so the reference's recorded decision is comparable too
        same = live.clone()
        ref_same = live & on_ref
        chain = [(tl, dbg["text_logits"].float()[:, 0, 0], 0.7, 25, nt, tt, dbg["text_token"], gold["sampled_text"][i])]
        for k in range(cfg.dep_q):
            chain.append((dl[k], dbg["dep_logits"][k].float()[:, 0, 0], 0.8, 250, na[k], at[k], dbg["audio_tokens"][:, k],
                          gold["sampled_audio"][i][:, k]))
        for lg, lo, temp, topk, nz, tok_g, tok_o, tok_r in chain:
            for b in range(B):
                if not same[b]:
                    ref_same[b] = False       # the oracle's logits no longer describe this row's sampler inputs
                    continue
                d = float((lg[b] - lo[b]).abs().max())
                ok = bool(sample_is_stable(lo[b:b + 1], temp, topk, nz[b:b + 1], d + 1e-6)[0])
                c["worst"] = max(c["worst"], d)
                c["decisions"] += 1
                c["stable"] += int(ok)
                if ref_same[b]:
                    c["ref_decisions"] += 1
                    if int(tok_g[b]) == int(tok_r[b]):
                        c["ref_equal"] += 1
                    else:
                        ref_same[b] = False
                        c["ref_unexcused"] += int(ok)
                if int(tok_g[b]) == int(tok_o[b]):
                    c["equal"] += 1
                else:
                    same[b] = False
                    c["unexcused"] += int(ok)
        on_ref &= ~live | ref_same            # a row stays on the reference's trajectory only if every decision of this step matched
        pos = (orc.offsets % orc.cache.shape[2])
        for b in range(B):
            if live[b]:
                orc.cache[b, 0, pos[b]] = tt[b]
                orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
    return c


@pytest.mark.parametrize("use_graph", [False, True])
def test_sampled_tokens_margin_aware_on_peaked_distributions(golden_dir, use_graph):
    """north_star: "sampled token ids under a fixed seed".  On peaked output distributions (scenarios.peaked_state_dict: what a
    trained model produces) every sampler decision is compared with the oracle's, fed the same Exp(1) draws: the ids must be
    EQUAL unless the decision is provably unstable under the logit difference actually observed for that row
    (tests/util.sample_is_stable: candidates closer than twice that difference may swap ranks and thereby noise values, scores
    move by at most 2 * diff / temp).  The same gate against the unmodified reference's own sampler decisions, recorded with torch's
    seeded CPU generator (tests/golden/lm_tiny_sampled_peaked.safetensors: every text / audio token as sampled, via the on_text /
    on_audio hooks): while a row's token history equals the reference's, each decision equals the reference's or is provably
    unstable (which includes exact bf16 ties, whose torch.topk order is unspecified)."""
    from moshi_b200.models import LMGen, LMModel
    cfg = tiny_lm_config()
    sd = scenarios.peaked_state_dict(cfg)
    gold = load_file(golden_dir / "lm_tiny_sampled_peaked.safetensors")
    lm = LMModel(cfg, sd, device="cuda")
    gen = LMGen(lm, use_sampling=True, temp=0.8, temp_text=0.7)
    gen.use_graph = use_graph
    B = scenarios.LM_B

    class Dev:
        def set_exec_mask(self, m):
            gen.set_exec_mask(m)

        def reset_streaming(self, m=None):
            gen.reset_streaming(m)

        def step(self, codes, nt, na):
            return gen.step(codes.cuda(), noise=gen.pack_noise(nt, na))

        def outputs(self):
            return (gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu(),
                    gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu(),
                    gen.read_buffer("text_token", torch.int64, (B,)).cpu(), gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu())

    with gen.streaming(B):
        c = _peaked_sampling_run(Dev(), sd, cfg, gold)
    print(f"peaked sampling (graph={use_graph}): {c['decisions']} sampler decisions compared, {c['stable']} provably stable under the "
          f"observed logit difference, {c['equal']} equal, {c['unexcused']} unexcused mismatches; against the reference's recorded "
          f"decisions: {c['ref_decisions']} compared, {c['ref_equal']} equal, {c['ref_unexcused']} unexcused; worst logit diff {c['worst']:.3e}")
    assert c["unexcused"] == 0 and c["ref_unexcused"] == 0
    assert c["stable"] > 0.4 * c["decisions"]            # the gate is not vacuous
    assert c["equal"] > 0.9 * c["decisions"]
    assert c["worst"] < 4 * LOGIT_ATOL              # logits are 4x larger than in the default scenario (bf16 ulp 0.06-0.125 at |x| 8-32)
    assert c["ref_decisions"] > 30
