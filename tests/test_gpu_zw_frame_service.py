"""GPU: ``DialogueService.step`` / ``b200_frame_step`` (host buffers in and out, one wait per frame) against the same frame
driven call by call through ``MimiModel.encode`` -> ``LMGen.step`` -> ``MimiModel.decode`` on twin models — the loop of
``server.py:120-147`` with the slot bookkeeping of ``batched_asr.py:138-215``.  Bit-exact: both paths launch the same
kernels in the same order on the same inputs."""
import numpy as np
import pytest
import torch

from moshi_b200.config import MimiConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict, synth_mimi_state_dict
from oracle import scenarios

pytestmark = pytest.mark.gpu


def _models():
    from moshi_b200.models import LMModel, MimiModel
    cfg = tiny_lm_config(card=2048)             # the LM reads and writes the codec's 2048-entry codebooks
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    msd = synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED)
    return cfg, LMModel(cfg, sd, device="cuda"), MimiModel(MimiConfig(), msd, device="cuda")


@pytest.mark.parametrize("sampling", [False, True, "internal"])
def test_frame_service_equals_call_by_call(sampling):
    """``sampling``: False = greedy; True = sampled with the caller's Exp(1) draws; "internal" = sampled with no noise passed
    (both pointers NULL), so each LM step draws its own, seeded from torch's generator when streaming starts."""
    from moshi_b200.models import LMGen
    from moshi_b200.serving import ACTIVE, NODATA, RESET, DialogueService
    B, steps = 4, 12
    internal = sampling == "internal"
    sampling = bool(sampling)
    cfg, lm_a, mimi_a = _models()
    _, lm_b, mimi_b = _models()
    torch.manual_seed(1234)
    svc = DialogueService(B, lm_a, mimi_a, use_sampling=sampling)
    gen = LMGen(lm_b, use_sampling=sampling, support_out_of_sync=True)
    torch.manual_seed(1234)
    gen.streaming_forever(B)
    mimi_b.streaming_forever(B)
    g = torch.Generator().manual_seed(7)
    active = torch.ones(B, dtype=torch.bool)
    npr = svc._lib.b200_lm_noise_per_row(lm_a._h)
    produced = not_greedy = 0
    for i in range(steps):
        pcm = 0.1 * torch.randn(B, 1, 1920, generator=g)
        noise = torch.empty(B, npr).exponential_(1, generator=g) if sampling and not internal else None
        updates = [9] * B                      # a positive marker: slot keeps its state (batched_asr.py:161-170)
        if i == 0:
            updates = [ACTIVE] * B
        if i == 3:
            updates[1] = NODATA
        if i == 6:
            updates[1] = ACTIVE
            updates[2] = RESET
        reset = torch.tensor([u == RESET for u in updates])
        for b, u in enumerate(updates):
            if u == NODATA:
                active[b] = False
            elif u in (ACTIVE, RESET):
                active[b] = True
        # ---- service
        pcm_out = np.zeros((B, 1920), dtype=np.float32)
        tok_out = np.zeros((B, cfg.dep_q + 1), dtype=np.int64)
        flags = np.zeros(B, dtype=np.uint8)
        svc.step(pcm.reshape(-1).numpy().copy(), pcm_out, tok_out, updates=updates, flags_out=flags,
                 noise=None if noise is None else noise.numpy().copy())
        # ---- call by call (what server.py / batched_asr.py do around the same handles)
        if reset.any():
            gen.reset_streaming(reset.cuda())
            mimi_b.reset_streaming(reset.cuda())
        gen.set_exec_mask(active.cuda())
        mimi_b.set_exec_mask(active.cuda())
        codes = mimi_b.encode(pcm.cuda())
        toks = gen.step(codes, noise=None if noise is None else noise.cuda())
        assert toks is not None
        ready = active.cuda() & (toks[:, :, 0] >= 0).all(dim=1)
        mimi_b.set_exec_mask(ready)
        want_pcm = mimi_b.decode(toks[:, 1:].clamp(min=0) * ready[:, None, None])
        ready = ready.cpu()
        assert np.array_equal(flags.astype(bool), ready.numpy()), (i, flags, ready)
        want_tok = toks[:, :, 0].cpu()
        if internal:             # tokens other than the argmax of their own logits: the step did sample
            tl = gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float()
            dl = gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float()
            tt = gen.read_buffer("text_token", torch.int64, (B,))
            at = gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B))
            not_greedy += int((tt != tl.argmax(-1)).sum()) + int((at != dl.argmax(-1)).sum())
        for b in range(B):
            if ready[b]:
                assert np.array_equal(tok_out[b], want_tok[b].numpy()), (i, b)
                assert np.array_equal(pcm_out[b], want_pcm[b, 0].cpu().numpy()), (i, b)
                produced += 1
            else:
                assert (pcm_out[b] == 0).all()
                assert (tok_out[b] < 0).any() or not active[b]
    assert produced >= B * (steps - 4)
    if internal:
        assert not_greedy > 0, "with no noise passed, every token was the greedy one"
    # warm-up rows: a reset slot is silent for max_delay frames again (lm.py:779-782)
    svc.close()


def test_frame_service_rejects_bad_buffers():
    from moshi_b200.serving import DialogueService
    cfg, lm, mimi = _models()
    svc = DialogueService(2, lm, mimi, use_sampling=False)
    good = np.zeros(2 * 1920, dtype=np.float32)
    with pytest.raises(AssertionError):
        svc.step(good[:100], np.zeros((2, 1920), np.float32), np.zeros((2, 9), np.int64))
    with pytest.raises(ValueError):
        svc.step(good, np.zeros((2, 1920), np.float32), np.zeros((2, 9), np.int64), updates=[-7, 0])
    svc.close()


def test_frame_service_against_the_oracle_pipeline():
    """The frame service against the ORACLE (not against the CUDA path itself): every frame, the CPU restatement of the
    reference runs the same three stages, each fed the GPU's own hand-off so that one excused flip does not make the rest
    incomparable: (1) ``MimiOracle.encode`` of the same PCM vs the codes the service handed to the LM (margin-aware RVQ
    comparison, no unexcused index), (2) ``LMOracle.step`` on those codes vs the service's logits / greedy tokens (tolerance +
    margin-aware ids), (3) ``MimiOracle.decode`` of the service's tokens vs the PCM it returned; with a paused and a
    recycled slot, and the decoder advancing only for rows that are past their delay warm-up (server.py:139-142)."""
    from moshi_b200.models import LMModel, MimiModel
    from moshi_b200.serving import ACTIVE, NODATA, RESET, DialogueService
    from oracle.lm import LMOracle, LMSpec
    from oracle.mimi import MimiOracle
    from tests.util import greedy_unexcused, rvq_mismatches
    B, steps = 4, 10
    mcfg = MimiConfig()
    cfg = tiny_lm_config(card=2048)
    sd = synth_lm_state_dict(cfg, seed=scenarios.LM_SEED)
    msd = synth_mimi_state_dict(mcfg, seed=scenarios.MIMI_SEED)
    svc = DialogueService(B, LMModel(cfg, sd, device="cuda"), MimiModel(mcfg, msd, device="cuda"), use_sampling=False)
    m_orc = MimiOracle(msd, mcfg)
    m_orc.streaming(B)
    l_orc = LMOracle(sd, LMSpec.from_config(cfg), use_sampling=False, tie_break="index")
    l_orc.streaming(B)
    g = torch.Generator().manual_seed(21)
    active = torch.ones(B, dtype=torch.bool)
    tol = 0.12          # 2048-way audio heads on the tiny model: measured worst 0.086
    code_bad = code_unexc = tok_bad = tok_unexc = tok_total = frames_out = 0
    worst_logit = worst_pcm = 0.0
    for i in range(steps):
        pcm = 0.1 * torch.randn(B, 1, 1920, generator=g)
        updates = [9] * B
        if i == 0:
            updates = [ACTIVE] * B
        if i == 3:
            updates[1] = NODATA
        if i == 5:
            updates[1] = ACTIVE
            updates[2] = RESET
        reset = torch.tensor([u == RESET for u in updates])
        for b, u in enumerate(updates):
            if u == NODATA:
                active[b] = False
            elif u in (ACTIVE, RESET):
                active[b] = True
        pcm_out = np.zeros((B, 1920), dtype=np.float32)
        tok_out = np.zeros((B, cfg.dep_q + 1), dtype=np.int64)
        flags = np.zeros(B, dtype=np.uint8)
        svc.step(pcm.reshape(-1).numpy().copy(), pcm_out, tok_out, updates=updates, flags_out=flags)
        gpu_codes = svc.read_buffer("codes_in", torch.int64, (B, 8)).cpu()
        # ---- oracle, stage by stage
        if reset.any():
            m_orc.reset_streaming(reset)
            l_orc.reset_streaming(reset)
        m_orc.set_exec_mask(active)
        l_orc.set_exec_mask(active)
        want_codes, margins = m_orc.quantize(m_orc.encode_to_latent(pcm), return_margins=True)
        bad, unexc = rvq_mismatches(gpu_codes[active][:, :, None], want_codes[active], margins[active])
        code_bad += bad
        code_unexc += unexc
        dbg = {}
        want = l_orc.step(gpu_codes[:, :, None], None, None, debug=dbg, support_out_of_sync=True)
        tl = svc.lm_gen.read_buffer("text_logits", torch.bfloat16, (B, cfg.text_card)).float().cpu()
        tlo = dbg["text_logits"].float()[:, 0, 0]
        worst_logit = max(worst_logit, (tl - tlo)[active].abs().max().item())
        tt = svc.lm_gen.read_buffer("text_token", torch.int64, (B,)).cpu()
        at = svc.lm_gen.read_buffer("audio_tokens", torch.int64, (cfg.dep_q, B)).cpu()
        m, u = greedy_unexcused(tt[active], dbg["text_token"][active], tlo[active], tol)
        tok_bad += m; tok_unexc += u; tok_total += int(active.sum())
        same = active & (tt == dbg["text_token"])
        dl = svc.lm_gen.read_buffer("dep_logits", torch.bfloat16, (cfg.dep_q, B, cfg.card)).float().cpu()
        for k in range(cfg.dep_q):
            if not same.any():
                break
            dlo = dbg["dep_logits"][k].float()[:, 0, 0]
            worst_logit = max(worst_logit, (dl[k] - dlo)[same].abs().max().item())
            m, u = greedy_unexcused(at[k][same], dbg["audio_tokens"][:, k][same], dlo[same], tol)
            tok_bad += m; tok_unexc += u; tok_total += int(same.sum())
            same = same & (at[k] == dbg["audio_tokens"][:, k])
        pos = (l_orc.offsets % l_orc.cache.shape[2])
        for b in range(B):                        # keep the oracle's token ring on the GPU's trajectory
            if active[b]:
                l_orc.cache[b, 0, pos[b]] = tt[b]
                l_orc.cache[b, 1:cfg.dep_q + 1, pos[b]] = at[:, b]
        # the re-aligned output of the step must be what the (synchronised) oracle ring now holds (lm.py:774-783)
        gd = l_orc.delays[:cfg.dep_q + 1]
        idx = (l_orc.offsets[:, None, None] - cfg.max_delay + gd[:, None]) % l_orc.cache.shape[2]
        want_out = l_orc.cache[:, :cfg.dep_q + 1].gather(2, idx)[:, :, 0]
        ready = active & (l_orc.offsets > cfg.max_delay)
        assert np.array_equal(flags.astype(bool), ready.numpy()), (i, flags, ready)
        assert np.array_equal(tok_out[ready.numpy()], want_out[ready].numpy()), i
        # ---- decoder: only ready rows advance
        m_orc.set_exec_mask(ready)
        want_pcm = m_orc.decode((torch.from_numpy(tok_out[:, 1:]).clamp(min=0) * ready[:, None])[:, :, None])
        for b in range(B):
            if ready[b]:
                worst_pcm = max(worst_pcm, float(np.abs(pcm_out[b] - want_pcm[b, 0].numpy()).max()))
                frames_out += 1
            else:
                assert (pcm_out[b] == 0).all()
    print(f"frame service vs oracle: RVQ codes mismatches {code_bad} (unexcused {code_unexc}); greedy ids compared {tok_total}, "
          f"mismatches {tok_bad} (unexcused {tok_unexc}); worst logit diff {worst_logit:.3e}; worst PCM diff {worst_pcm:.3e} over "
          f"{frames_out} decoded frames")
    assert code_unexc == 0 and tok_unexc == 0
    assert worst_logit < tol and worst_pcm < 5e-4
    assert frames_out >= B * (steps - 4)
    svc.close()
