"""GPU: the batched speech-to-text service (``serving.ASRService`` / ``b200_asr_step``) against ``ASRService`` of
``rust/moshi-server/batched_asr.py`` restated over this library's ``MimiModel`` + ``LMGen`` (the same kernels, so every output
must be identical), and against the oracle."""
import dataclasses
import json
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from moshi_b200.config import LMConfig, MimiConfig, tiny_lm_config
from moshi_b200.synth import synth_lm_state_dict, synth_mimi_state_dict
from oracle import scenarios

pytestmark = pytest.mark.gpu

NODATA, ACTIVE, RESET = 0, -1, -2
FLAG_SENTINEL, TOKEN_SENTINEL, HEAD_SENTINEL = 0xAB, 0xDEADBEEF, -7.0


# ---- batched_asr.py:85-213, line by line over the library's classes ----------------------------------------------------------
@dataclass
class ClientState:
    is_complete: bool = False
    active: bool = False
    offset: int = 0
    real_end: int = 0

    def reset(self) -> None:
        self.active = False
        self.is_complete = False
        self.offset = 0
        self.real_end = 0


class TwinASRService:
    def __init__(self, batch_size, lm, mimi, asr_delay_in_tokens, temp=0.0, device="cuda"):
        from moshi_b200.models import LMGen
        self.batch_size, self.lm, self.mimi, self.asr_delay_in_tokens = batch_size, lm, mimi, asr_delay_in_tokens
        self.device = device
        self.lm_gen = LMGen(self.lm, temp_text=temp)
        self.lm_gen.streaming_forever(self.batch_size)
        self.mimi.streaming_forever(self.batch_size)
        self.clients = [ClientState() for _ in range(self.batch_size)]
        for _ in range(3):
            self.mimi.set_exec_mask(torch.ones(self.batch_size, dtype=torch.bool))
            self.lm_gen.set_exec_mask(torch.ones(self.batch_size, dtype=torch.bool))
            batch_zeros = torch.zeros((self.batch_size, 1, self.mimi.frame_size), dtype=torch.float32, device=self.device)
            audio_tokens = self.mimi.encode(batch_zeros)
            frame = self.lm_gen.step(audio_tokens)
            assert frame is not None

    @torch.no_grad()
    def step(self, batch_pcm, flags_out, tokens_out, extra_heads, updates) -> bool:
        reset_mask = torch.zeros(self.batch_size, dtype=torch.bool)
        for batch_idx, update in enumerate(updates):
            if update == NODATA:
                self.clients[batch_idx].active = False
                flags_out[batch_idx] = 0
            if update == ACTIVE:
                self.clients[batch_idx].active = True
                flags_out[batch_idx] = 1
            if update == RESET:
                self.clients[batch_idx].reset()
                flags_out[batch_idx] = 1
                reset_mask[batch_idx] = True
                self.clients[batch_idx].active = True
            if update > 0:
                self.clients[batch_idx].is_complete = True
                flags_out[batch_idx] = 2
                self.clients[batch_idx].real_end = self.clients[batch_idx].offset + update + self.asr_delay_in_tokens + 2
        exec_mask = torch.tensor([client.active for client in self.clients], dtype=torch.bool, device=self.device)
        need_reset = reset_mask.any()
        reset_mask = reset_mask.to(self.device)
        skip_exec = not exec_mask.any()
        if need_reset:
            self.lm_gen.reset_streaming(reset_mask=reset_mask)
            self.mimi.reset_streaming(reset_mask=reset_mask)
        if skip_exec:
            return False
        self.lm_gen.set_exec_mask(exec_mask)
        self.mimi.set_exec_mask(exec_mask)
        batch_pcm = torch.from_numpy(batch_pcm).to(self.device).view(self.batch_size, self.mimi.frame_size).unsqueeze(1)
        audio_tokens = self.mimi.encode(batch_pcm)
        text_tokens, extra_heads_list = self.lm_gen.step_with_extra_heads(audio_tokens)
        extra_heads_stacked = torch.stack(extra_heads_list, dim=0)[:, :, 0, 0]
        extra_heads[:, :] = extra_heads_stacked.transpose(0, 1).to(torch.float32).cpu().numpy()
        tokens_out[:] = text_tokens.cpu().numpy()[:, 0, 0]
        for batch_idx, client in enumerate(self.clients):
            if client.active:
                client.offset += 1
                if client.is_complete and client.offset >= client.real_end:
                    client.active = False
                    flags_out[batch_idx] = 4
        return True

    def close(self):
        self.lm_gen._stop()
        self.mimi._stop()


# ---- models and schedules -----------------------------------------------------------------------------------------------------
def _stt_config(**over) -> LMConfig:
    return LMConfig.from_dict(dict(scenarios.stt_reference_kwargs(), card=2048, **over))     # the codec's 2048-entry codebooks


def _mid_stt_config() -> LMConfig:
    """An STT-shaped LM of serving geometry in every dimension the kernels tile by: 32 user codebooks, no depformer, head dim
    128, 4 extra heads of 6 (the voice-activity heads the Rust server reads)."""
    return tiny_lm_config(dim=512, num_heads=4, num_layers=2, text_card=4000, n_q=32, dep_q=0, card=2048, context=40,
                          delays=[0] * 33, extra_heads_num_heads=4, extra_heads_dim=6)


def _pair(cfg, sd, msd, mcfg):
    from moshi_b200.models import LMModel, MimiModel
    return LMModel(cfg, sd, device="cuda"), MimiModel(mcfg, msd, device="cuda")


def _schedule_tiny(i: int, B: int) -> list[int]:
    """40 frames over 5 slots: an idle start, resets and a slot used without one (post-warm-up state), a pause, a marker that
    counts down to its end of stream, a repeated marker, a marker on a paused slot, an update value the reference ignores, a
    reset after an end of stream, and idle frames later on."""
    assert B == 5
    if i < 2 or i in (33, 34):
        return [NODATA] * B
    u = [ACTIVE] * B
    if i == 2:
        u = [RESET, RESET, ACTIVE, NODATA, NODATA]
    if i < 5:
        u[3] = u[4] = NODATA
    if i == 5:
        u[3] = RESET
        u[4] = RESET
    if i in (8, 9):
        u[1] = NODATA                      # pause
    if i == 12:
        u[0] = 3                           # end of stream: 3 more frames + delay + 2
    if 12 + 3 + 4 + 2 <= i < 30:
        u[0] = NODATA                      # after its end of stream (frame 20) the server stops sending
    if i == 14:
        u[4] = 6
    if i == 16:
        u[4] = 2                           # repeated marker: real_end recomputed from the current offset
    if i in (20, 21):
        u[3] = NODATA
    if i == 21:
        u[3] = 1                           # marker on a paused slot: flag 2, no countdown until it runs again
    if i == 25:
        u[2] = -5                          # not an UpdateFlags value: nothing written, nothing changes
    if i == 30:
        u[0] = RESET                       # a new session in the slot that ended
    if i == 35:
        u = [NODATA, NODATA, 4, NODATA, NODATA]     # a marker while nothing runs
    if i == 36:
        u = [ACTIVE, NODATA, ACTIVE, RESET, NODATA]
    return u


def _schedule_serving(i: int, B: int) -> list[int]:
    u = [ACTIVE] * B
    if i == 0:
        u = [RESET] * B
        u[-1] = ACTIVE                     # one slot used without a reset
    if i == 4:
        u[B - 1] = 2                       # one end of stream: EOS once offset reaches 4 + 2 + delay(2) + 2, after frame 9
    if i >= 10:
        u[B - 1] = NODATA
    if i == 7:
        u[1] = RESET
    if i in (9, 10):
        u[0] = NODATA
    return u


def _run_against_twin(svc, twin, B, frames, schedule, n_heads, seed):
    g = torch.Generator().manual_seed(seed)
    flags = [np.full(B, FLAG_SENTINEL, np.uint8) for _ in range(2)]
    toks = [np.full(B, TOKEN_SENTINEL, np.uint32) for _ in range(2)]
    heads = [np.full((B, n_heads), HEAD_SENTINEL, np.float32) for _ in range(2)]
    ran_frames = eos = markers = 0
    for i in range(frames):
        pcm = (0.1 * torch.randn(B * 1920, generator=g)).numpy()
        upd = schedule(i, B)
        ran = svc.step(pcm.copy(), flags[0], toks[0], heads[0], list(upd))
        ran_twin = twin.step(pcm.copy(), flags[1], toks[1], heads[1], list(upd))
        assert ran == ran_twin, i
        assert np.array_equal(flags[0], flags[1]), (i, upd, flags[0], flags[1])
        assert np.array_equal(toks[0], toks[1]), (i, toks[0], toks[1])
        assert np.array_equal(heads[0], heads[1]), (i, np.abs(heads[0] - heads[1]).max())
        off = svc.read_buffer("offset", torch.int64, (B,)).cpu().tolist()
        assert off == [c.offset for c in twin.clients], (i, off)
        ran_frames += ran
        eos += int((flags[0] == 4).sum())
        markers += int((flags[0] == 2).sum())
    return ran_frames, eos, markers


# ---- 1. bit-exact against the reference's loop ----------------------------------------------------------------------------------
@pytest.mark.parametrize("temp", [0.0, 0.8])
def test_asr_service_equals_the_reference_loop(temp):
    from moshi_b200.serving import ASRService
    B, frames, delay = 5, 40, 4
    cfg = _stt_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.STT_SEED)
    mcfg = MimiConfig()
    msd = synth_mimi_state_dict(mcfg, seed=scenarios.MIMI_SEED)
    lm_a, mimi_a = _pair(cfg, sd, msd, mcfg)
    lm_b, mimi_b = _pair(cfg, sd, msd, mcfg)
    torch.manual_seed(1234)
    svc = ASRService(B, lm_a, mimi_a, asr_delay_in_tokens=delay, temp=temp)
    torch.manual_seed(1234)
    twin = TwinASRService(B, lm_b, mimi_b, asr_delay_in_tokens=delay, temp=temp)
    ran, eos, markers = _run_against_twin(svc, twin, B, frames, _schedule_tiny, cfg.extra_heads_num_heads, seed=3)
    print(f"asr service vs reference loop (temp {temp}): {ran}/{frames} frames ran, {markers} marker flags, {eos} end-of-stream flags")
    assert ran == frames - 5 and eos >= 3 and markers >= 5
    svc.close()
    twin.close()


# ---- 2. 32 codebooks at serving batch -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [3, 64])
def test_asr_service_32_codebooks_at_serving_batch(B):
    from moshi_b200.serving import ASRService
    cfg = _mid_stt_config()
    sd = synth_lm_state_dict(cfg, seed=11)
    mcfg = MimiConfig(num_codebooks=32)
    msd = synth_mimi_state_dict(mcfg, seed=scenarios.MIMI_SEED)
    lm_a, mimi_a = _pair(cfg, sd, msd, mcfg)
    lm_b, mimi_b = _pair(cfg, sd, msd, mcfg)
    torch.manual_seed(5)
    svc = ASRService(B, lm_a, mimi_a, asr_delay_in_tokens=2)
    torch.manual_seed(5)
    twin = TwinASRService(B, lm_b, mimi_b, asr_delay_in_tokens=2)
    ran, eos, _ = _run_against_twin(svc, twin, B, 20, _schedule_serving, 4, seed=8)
    assert svc.read_buffer("codes_in", torch.int64, (B, 32)).max() < 2048
    print(f"asr service at {B} slots, 32 codebooks: {ran} frames bit-exact, {eos} end-of-stream flags")
    assert ran == 20 and eos == 1
    svc.close()
    twin.close()


# ---- 3. against the oracle ------------------------------------------------------------------------------------------------------
def test_asr_service_against_the_oracle():
    """The service against the CPU restatement of the reference, stage by stage and fed the service's own hand-off each frame:
    ``MimiOracle.encode`` vs the codes the service gave the LM (margin-aware RVQ), ``LMOracle.step_with_extra_heads`` on those
    codes vs the text tokens (margin-aware greedy ids) and the extra heads (8e-3, the STT gate), with the client state machine
    restated on the host deciding which rows execute."""
    from moshi_b200.serving import ASRService
    from oracle.lm import LMOracle, LMSpec
    from oracle.mimi import MimiOracle
    from tests.util import greedy_unexcused, rvq_mismatches
    B, frames, delay = 4, 12, 1
    cfg = _stt_config()
    sd = synth_lm_state_dict(cfg, seed=scenarios.STT_SEED)
    mcfg = MimiConfig()
    msd = synth_mimi_state_dict(mcfg, seed=scenarios.MIMI_SEED)
    lm, mimi = _pair(cfg, sd, msd, mcfg)
    svc = ASRService(B, lm, mimi, asr_delay_in_tokens=delay)
    spec = dataclasses.replace(LMSpec.from_config(cfg), extra_heads_num_heads=cfg.extra_heads_num_heads, extra_heads_dim=cfg.extra_heads_dim)
    m_orc = MimiOracle(msd, mcfg)
    m_orc.streaming(B)
    l_orc = LMOracle(sd, spec, use_sampling=False, tie_break="index")
    l_orc.streaming(B)
    clients = [ClientState() for _ in range(B)]
    g = torch.Generator().manual_seed(17)
    flags = np.zeros(B, np.uint8)
    toks = np.zeros(B, np.uint32)
    heads = np.zeros((B, cfg.extra_heads_num_heads), np.float32)
    tol = 0.08
    code_bad = code_unexc = tok_bad = tok_unexc = rows = 0
    worst_head = 0.0
    for i in range(frames):
        upd = [RESET] * B if i == 0 else [ACTIVE] * B
        if i in (3, 4):
            upd[1] = NODATA
        if i == 5:
            upd[2] = 1
        if i == 7:
            upd[3] = RESET
        pcm = 0.1 * torch.randn(B, 1, 1920, generator=g)
        ran = svc.step(pcm.reshape(-1).numpy().copy(), flags, toks, heads, upd)
        reset = torch.tensor([u == RESET for u in upd])
        for b, u in enumerate(upd):
            if u == NODATA:
                clients[b].active = False
            elif u in (ACTIVE, RESET):
                if u == RESET:
                    clients[b].reset()
                clients[b].active = True
            elif u > 0:
                clients[b].is_complete = True
                clients[b].real_end = clients[b].offset + u + delay + 2
        active = torch.tensor([c.active for c in clients])
        assert ran == bool(active.any())
        if reset.any():
            m_orc.reset_streaming(reset)
            l_orc.reset_streaming(reset)
        m_orc.set_exec_mask(active)
        l_orc.set_exec_mask(active)
        gpu_codes = svc.read_buffer("codes_in", torch.int64, (B, 8)).cpu()
        want_codes, margins = m_orc.quantize(m_orc.encode_to_latent(pcm), return_margins=True)
        bad, unexc = rvq_mismatches(gpu_codes[active][:, :, None], want_codes[active], margins[active])
        code_bad += bad
        code_unexc += unexc
        dbg = {}
        want, want_heads = l_orc.step_with_extra_heads(gpu_codes[:, :, None], debug=dbg)
        got = torch.from_numpy(toks.astype(np.int64).astype(np.int32)).long()      # uint32 wrap of -2 back to a signed id
        assert (got[~active] == -2).all()
        m, u = greedy_unexcused(got[active], dbg["text_token"][active], dbg["text_logits"].float()[:, 0, 0][active], tol)
        tok_bad += m
        tok_unexc += u
        rows += int(active.sum())
        want_h = torch.stack([h[:, 0, 0].float() for h in want_heads], dim=1)        # [B, n]
        worst_head = max(worst_head, float((torch.from_numpy(heads) - want_h)[active].abs().max()))
        pos = l_orc.offsets % l_orc.cache.shape[2]
        for b in range(B):                 # keep the oracle's token ring on the service's trajectory
            if active[b]:
                l_orc.cache[b, 0, pos[b]] = int(got[b])
        for b, c in enumerate(clients):
            if c.active:
                c.offset += 1
                if c.is_complete and c.offset >= c.real_end:
                    c.active = False
                    assert flags[b] == 4, (i, b, flags)
    print(f"asr service vs oracle: RVQ mismatches {code_bad} (unexcused {code_unexc}); text ids compared {rows}, mismatches "
          f"{tok_bad} (unexcused {tok_unexc}); worst extra-head probability diff {worst_head:.3e}")
    assert code_unexc == 0 and tok_unexc == 0
    assert worst_head < 8e-3 and rows >= B * (frames - 4)
    svc.close()


# ---- 4. refusals -----------------------------------------------------------------------------------------------------------------
def _handles_are_free(lm, mimi, B=2):
    """Both handles can stream again: a refused service left neither streaming nor holding anything of its own."""
    from moshi_b200.models import LMGen
    assert not mimi.is_streaming
    gen = LMGen(lm, use_sampling=False)
    gen.streaming_forever(B)
    mimi.streaming_forever(B)
    gen._stop()
    mimi._stop()


def test_asr_service_refusals():
    import ctypes as C

    from moshi_b200 import _lib
    from moshi_b200.models import LMGen, LMModel, MimiModel
    from moshi_b200.serving import ASRService
    mcfg = MimiConfig()
    msd = synth_mimi_state_dict(mcfg, seed=scenarios.MIMI_SEED)
    mimi = MimiModel(mcfg, msd, device="cuda")
    # a dialogue LM (depformer)
    dial = tiny_lm_config(card=2048)
    lm_dial = LMModel(dial, synth_lm_state_dict(dial, seed=1), device="cuda")
    with pytest.raises(ValueError, match="dep_q"):
        ASRService(2, lm_dial, mimi)
    _handles_are_free(lm_dial, mimi)
    # an STT LM with delays
    delayed = _stt_config(delays=[0] + [1] * 8)
    lm_del = LMModel(delayed, synth_lm_state_dict(delayed, seed=2), device="cuda")
    with pytest.raises(ValueError, match="delay"):
        ASRService(2, lm_del, mimi)
    _handles_are_free(lm_del, mimi)
    # a codec with fewer codebooks than the LM reads
    cfg = _stt_config()
    lm = LMModel(cfg, synth_lm_state_dict(cfg, seed=3), device="cuda")
    mimi4 = MimiModel(MimiConfig(num_codebooks=4), synth_mimi_state_dict(MimiConfig(num_codebooks=4), seed=scenarios.MIMI_SEED),
                      device="cuda")
    with pytest.raises(ValueError, match="codebooks"):
        ASRService(2, lm, mimi4)
    _handles_are_free(lm, mimi4)
    # handles streaming another batch (the C ABI: the Python service starts both itself)
    lib = _lib.lib()
    gen = LMGen(lm, use_sampling=False)
    gen.streaming_forever(3)
    mimi.streaming_forever(2)
    h = C.c_void_p()
    rc = lib.b200_asr_create(mimi._h, lm._h, 2, 32, _lib.current_stream(lm.device), C.byref(h))
    assert rc == _lib.B200_ERR_INVALID and b"batch" in lib.b200_last_error() and not h.value
    gen._stop()
    mimi._stop()
    # wrongly shaped buffers
    svc = ASRService(2, lm, mimi)
    pcm = np.zeros(2 * 1920, np.float32)
    ok = dict(flags_out=np.zeros(2, np.uint8), tokens_out=np.zeros(2, np.uint32), extra_heads=np.zeros((2, 2), np.float32))
    bad = [dict(batch_pcm=pcm[:100]), dict(flags_out=np.zeros(2, np.int32)), dict(flags_out=np.zeros(3, np.uint8)),
           dict(tokens_out=np.zeros(3, np.uint32)), dict(tokens_out=np.zeros(2, np.float32)),
           dict(extra_heads=np.zeros((2, 4), np.float32)), dict(extra_heads=np.zeros((2, 2), np.float64)), dict(updates=[ACTIVE])]
    for over in bad:
        kw = dict(batch_pcm=pcm, updates=[ACTIVE, ACTIVE], **ok)
        kw.update(over)
        with pytest.raises(AssertionError):
            svc.step(kw["batch_pcm"], kw["flags_out"], kw["tokens_out"], kw["extra_heads"], kw["updates"])
    assert svc.step(pcm, ok["flags_out"], ok["tokens_out"], ok["extra_heads"], [ACTIVE, NODATA])
    svc.close()
    _handles_are_free(lm, mimi)


# ---- the drop-in script ---------------------------------------------------------------------------------------------------------
def test_batched_asr_script_init_from_checkpoint_files(tmp_path):
    """``moshi_b200/batched_asr.py`` loaded the way the Rust server loads its script (from source, under another module name):
    ``init(batch_size, config)`` builds the service from local checkpoint files, unknown keys ignored."""
    import importlib.util
    from pathlib import Path

    from safetensors.torch import save_file
    cfg = _stt_config()
    save_file({k: v.contiguous() for k, v in synth_lm_state_dict(cfg, seed=4).items()}, str(tmp_path / "stt.safetensors"))
    save_file({k: v.contiguous() for k, v in synth_mimi_state_dict(MimiConfig(), seed=5).items()}, str(tmp_path / "mimi.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps(dict(scenarios.stt_reference_kwargs(), card=2048, model_type="stt",
                                                          mimi_name="mimi.safetensors", lm_gen_config={"temp": 0.0})))
    script = Path(__file__).resolve().parent.parent / "moshi_b200" / "batched_asr.py"
    spec = importlib.util.spec_from_file_location("foo", script)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    svc = mod.init(3, {"moshi_weight": str(tmp_path / "stt.safetensors"), "mimi_weight": str(tmp_path / "mimi.safetensors"),
                       "config_path": str(tmp_path / "config.json"), "tokenizer": str(tmp_path / "tok.model"),
                       "log_folder": str(tmp_path / "logs"), "asr_delay_in_tokens": 2, "debug": True, "text_tokenizer_file": "x"})
    assert (tmp_path / "logs").is_dir() and svc.mimi.num_codebooks == 8 and svc.asr_delay_in_tokens == 2
    flags, toks, heads = np.zeros(3, np.uint8), np.zeros(3, np.uint32), np.zeros((3, 2), np.float32)
    for i in range(6):                     # slot 1: marker at offset 1, end of stream once its offset reaches 1 + 1 + 2 + 2
        upd = [RESET, ACTIVE, NODATA] if i == 0 else [ACTIVE, 1 if i == 1 else ACTIVE, NODATA]
        assert svc.step(np.zeros(3 * 1920, np.float32), flags, toks, heads, upd)
        assert flags.tolist() == [1, 4 if i == 5 else 2 if i == 1 else 1, 0], (i, flags)
    assert (heads[:2] > 0).all() and (toks[2] == np.uint32(2 ** 32 - 2))
    svc.close()
