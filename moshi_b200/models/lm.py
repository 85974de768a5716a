"""``LMModel`` / ``LMGen`` with the reference's public surface, backed by the sm_90a library.

Mirrors ``moshi/moshi/models/lm.py``: ``LMModel`` exposes the attributes callers read
(``dep_q, n_q, card, text_card, delays, device, dtype, num_codebooks, condition_provider, fuser, ...``,
lm.py:248-295) and owns the weights on the device; ``LMGen`` (lm.py:555-850) owns the streaming state and runs one
``step`` per 80 ms frame, including classifier-free guidance (lm.py:596-604, 646-662, 714-732, 820-833), conditioning by
sum (lm.py:616-626), cross-attention conditioning of the temporal layers (lm.py:616-651, transformer.py:727-732, 779-798),
forced audio tokens (lm.py:751-755) and the STT models' extra heads (lm.py:793-807).

Sampling noise: the reference draws ``Exp(1)`` from torch's generator inside ``sample_token`` (sampling.py:44).  Here
the step draws it itself (a Philox stream inside the step's CUDA graph, seeded once per session from torch's CPU
generator, so ``torch.manual_seed`` still makes a run reproducible) unless the caller passes ``noise=`` explicitly,
which is how the parity tests feed the reference's own draws.
"""
from __future__ import annotations

import ctypes as C
import typing as tp
from contextlib import ExitStack
from types import SimpleNamespace

import torch

from .. import _lib
from ..conditioners import ConditionFuser, ConditionProvider, ConditionTensors, build_conditioning
from ..config import LMConfig
from .state_dict import candle_refusal, normalize_lm_state_dict

_TORCH_DTYPES = {_lib.B200_F32: torch.float32, _lib.B200_BF16: torch.bfloat16, _lib.B200_F16: torch.float16,
                 _lib.B200_I64: torch.int64, _lib.B200_U8: torch.uint8, _lib.B200_I32: torch.int32}


def _config_struct(cfg: LMConfig) -> _lib.LMConfigC:
    c = _lib.LMConfigC()
    c.dim, c.text_card, c.n_q, c.dep_q, c.card = cfg.dim, cfg.text_card, cfg.n_q, cfg.dep_q, cfg.card
    c.num_heads, c.num_layers, c.ffn_hidden, c.context = cfg.num_heads, cfg.num_layers, cfg.ffn_hidden, cfg.context
    c.max_period = cfg.max_period
    c.depformer_dim, c.depformer_num_heads = cfg.depformer_dim, cfg.depformer_num_heads
    c.depformer_num_layers, c.depformer_ffn_hidden = cfg.depformer_num_layers, cfg.depformer_ffn_hidden
    for i, d in enumerate(cfg.delays):
        c.delays[i] = d
    c.quantize = int(bool(cfg.quantize))
    c.extra_heads_num_heads, c.extra_heads_dim = cfg.extra_heads_num_heads, cfg.extra_heads_dim
    return c


class LMModel:
    """Moshi Temporal + Depth transformer weights on one GPU.  Construct via ``loaders.get_moshi_lm``."""

    def __init__(self, cfg: LMConfig, tensors: tp.Iterable[tuple[str, torch.Tensor]] | tp.Mapping[str, torch.Tensor],
                 device: torch.device | str = "cuda", dtype: torch.dtype = torch.bfloat16):
        cfg.check_supported()
        if dtype != torch.bfloat16:
            raise ValueError("the GPU LM path computes in bfloat16 (reference default, loaders.py:370)")
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("moshi_b200.LMModel runs on a CUDA device only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.dtype = dtype
        # attributes read by callers (lm.py:119-160, 248-295)
        self.n_q, self.dep_q, self.card, self.text_card = cfg.n_q, cfg.dep_q, cfg.card, cfg.text_card
        self.delays = list(cfg.delays)
        self.dim = cfg.dim
        self.context = cfg.context
        self.existing_text_padding_id = cfg.existing_text_padding_id
        self.condition_provider: ConditionProvider | None = None
        self.fuser: ConditionFuser | None = None
        self.depformer = True if cfg.dep_q > 0 else None          # lm.py:219-222: None for the no-depformer (STT) models
        self.extra_heads: list = [None] * cfg.extra_heads_num_heads
        self.training = False
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        items = tensors.items() if isinstance(tensors, tp.Mapping) else tensors
        host_side: dict[str, torch.Tensor] = {}       # conditioner weights stay with the Python-side provider
        with torch.cuda.device(self.device):
            _lib.check(self._lib.b200_lm_create(C.byref(_config_struct(cfg)), C.byref(self._h)))
            if cfg.cross_attention:
                _lib.check(self._lib.b200_lm_set_cross_attention(self._h, 1))
            if cfg.depformer_weights_per_step_schedule is not None:
                sched = cfg.depformer_weights_per_step_schedule
                _lib.check(self._lib.b200_lm_set_depformer_schedule(self._h, (C.c_int * len(sched))(*sched), len(sched)))
            if cfg.depformer_low_rank_embeddings is not None:
                _lib.check(self._lib.b200_lm_set_depformer_low_rank(self._h, cfg.depformer_low_rank_embeddings))
            for name, t in items:
                if name.startswith("condition_provider."):
                    host_side[name] = t.detach()
                    continue
                why = candle_refusal(cfg, name)
                if why is not None:
                    raise ValueError(why)
                for n2, t2 in normalize_lm_state_dict({name: t}).items():
                    # a q8 checkpoint stores a QLinear as `weight` int8 + `weight_scb` float32, and the scale must stay float32
                    # (utils/quantize.py:13-35; the reference's loader casts it with the rest, loaders.py:415-421, and then fails)
                    if t2.dtype == torch.int8:
                        want = torch.int8
                    elif n2.endswith(".weight_scb"):
                        want = torch.float32
                    else:
                        want = torch.bfloat16
                    t2 = t2.detach().to(device=self.device, dtype=want).contiguous()
                    shape = (C.c_int64 * t2.dim())(*t2.shape)
                    _lib.check(self._lib.b200_lm_load_tensor(self._h, n2.encode(), _lib.ptr(t2), _lib.dtype_code(want),
                                                             t2.dim(), shape))
                    del t2
            _lib.check(self._lib.b200_lm_finalize(self._h))
        if cfg.conditioners:
            self.condition_provider, self.fuser = build_conditioning(cfg.conditioners, cfg.fuser, cfg.dim, host_side, self.device,
                                                                     cfg.cross_attention)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self._lib.b200_lm_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    @property
    def num_codebooks(self) -> int:
        return self.n_q + 1

    @property
    def num_audio_codebooks(self) -> int:
        return self.n_q

    @property
    def audio_offset(self) -> int:
        return 1

    @property
    def initial_token_id(self) -> int:
        return self.card

    @property
    def text_initial_token_id(self) -> int:
        return self.text_card

    @property
    def text_padding_token_id(self) -> int:
        return self.existing_text_padding_id

    @property
    def zero_token_id(self) -> int:
        return -1

    @property
    def ungenerated_token_id(self) -> int:
        return -2

    def eval(self) -> "LMModel":
        return self


class LMGen:
    """``LMGen`` (lm.py:555-850)."""

    def __init__(self, lm_model: LMModel, use_sampling: bool = True, temp: float = 0.8, temp_text: float = 0.7,
                 top_k: int = 250, top_k_text: int = 25, cfg_coef: float = 1., check: bool = False,
                 condition_tensors: ConditionTensors | None = None, on_text_hook=None, on_text_logits_hook=None,
                 on_audio_hook=None, support_out_of_sync: bool = False, cfg_is_masked_until: list[int] | None = None,
                 cfg_is_no_text: bool = False):
        self.lm_model = lm_model
        self.use_sampling, self.temp, self.temp_text = use_sampling, temp, temp_text
        self.top_k, self.top_k_text = top_k, top_k_text
        self.cfg_coef = cfg_coef
        self.check = check
        self.max_delay = max(lm_model.delays)
        self.delays_cuda = torch.tensor(lm_model.delays, device=lm_model.device, dtype=torch.long)
        self.condition_tensors = condition_tensors
        self.on_text_hook, self.on_text_logits_hook, self.on_audio_hook = on_text_hook, on_text_logits_hook, on_audio_hook
        self.support_out_of_sync = support_out_of_sync
        self.cfg_is_masked_until = cfg_is_masked_until
        self.cfg_is_no_text = cfg_is_no_text
        if self.cfg_coef != 1.:                                      # lm.py:600-603
            if not self.cfg_is_no_text and not self.cfg_is_masked_until:
                assert self.lm_model.fuser is not None, "Model has no fuser, cannot do CFG."
                assert self.condition_tensors, "Missing condition tensors for CFG."
        self._lib = lm_model._lib
        self._h = lm_model._h
        self._batch: int | None = None
        self._streaming_state = None      # truthy while streaming (callers test `lm_gen._streaming_state`)
        self._pushed_sampling: tuple | None = None
        self._stream: int | None = None
        self.use_graph = True
        # "bf16" = the reference's ring; "fp8_e4m3" / "int8" = opt-in extensions outside the reference's numerics (half the ring)
        self.kv_dtype = "bf16"
        # slots per temporal KV ring; None = the model's context (the reference's RingKVCache).  A pool of sessions younger than
        # `kv_capacity` frames holds the same keys in kv_capacity / context of the memory; stepping past it raises error flag 4
        self.kv_capacity: int | None = None
        # paged temporal KV rings: the rings of all model rows share a pool of `kv_pool_frames` slots in pages of `kv_page_slots`;
        # a row takes pages as its fill grows and returns them on reset (None = one full ring per row).  Same numerics, bit for bit
        self.kv_pool_frames: int | None = None
        self.kv_page_slots = 64
        # per-session sampling settings (set_session_sampling): the length of each session's text-history ring in [1, 1024], or
        # None = every session samples with the handle-wide values above
        self.session_sampling: int | None = None

    # ---- plumbing ---------------------------------------------------------------------------------
    def _device(self):
        return torch.cuda.device(self.lm_model.device)

    def _push_sampling(self) -> None:
        """The reference reads use_sampling / temp / temp_text on every step (lm.py:735-741): re-push when they change."""
        cur = (int(self.use_sampling), float(self.temp), float(self.temp_text), int(self.top_k), int(self.top_k_text))
        if cur != self._pushed_sampling:
            _lib.check(self._lib.b200_lm_set_sampling(self._h, *cur))
            self._pushed_sampling = cur

    def _sync_stream(self) -> None:
        """Work is ordered on torch's current stream of the model's device, like the reference's ops would be."""
        s = torch.cuda.current_stream(self.lm_model.device).cuda_stream
        if s != self._stream:
            _lib.check(self._lib.b200_lm_set_stream(self._h, C.c_void_p(s)))
            self._stream = s

    # ---- streaming protocol ----------------------------------------------------------------------
    @property
    def is_streaming(self) -> bool:
        return self._batch is not None

    def _start(self, batch_size: int) -> None:
        assert self._batch is None, "lm_gen is already streaming!"
        lm, dev = self.lm_model, self.lm_model.device
        # lm.py:613-627: the sum- and cross-fused conditions, cast to the model dtype
        condition_sum = condition_cross = None
        if lm.fuser is None:
            assert not self.condition_tensors
        else:
            assert self.condition_tensors is not None
            condition_sum = lm.fuser.get_sum(self.condition_tensors)
            if condition_sum is not None:
                condition_sum = condition_sum.to(device=dev, dtype=lm.dtype)
            condition_cross = lm.fuser.get_cross(self.condition_tensors)
            if condition_cross is not None:
                condition_cross = condition_cross.to(device=dev, dtype=lm.dtype)
        model_batch = batch_size * 2 if self.cfg_coef != 1. else batch_size
        if condition_sum is not None:
            assert condition_sum.shape[0] == model_batch, "cfg requires 2x more conditions."     # lm.py:648-649
        if condition_cross is not None:
            assert condition_cross.shape[0] == model_batch, "cfg requires 2x more conditions."   # lm.py:650-651
        # transformer.py:786: every cross-attention layer needs its source
        assert condition_cross is not None or not lm.cfg.cross_attention, "a cross-attention LM needs cross condition tensors"
        with self._device():
            self._pushed_sampling = None
            self._push_sampling()
            _lib.check(self._lib.b200_lm_set_graph(self._h, int(self.use_graph)))
            kinds = {"bf16": 0, "fp8_e4m3": 1, "int8": 2}
            if self.kv_dtype not in kinds:
                raise ValueError(f"kv_dtype {self.kv_dtype!r}: expected one of {sorted(kinds)}")
            _lib.check(self._lib.b200_lm_set_kv_dtype(self._h, kinds[self.kv_dtype]))
            _lib.check(self._lib.b200_lm_set_kv_capacity(self._h, int(self.kv_capacity or 0)))
            _lib.check(self._lib.b200_lm_set_kv_pool(self._h, int(self.kv_pool_frames or 0), int(self.kv_page_slots)))
            _lib.check(self._lib.b200_lm_set_session_sampling(self._h, int(self.session_sampling or 0)))
            until = None
            if self.cfg_coef != 1. and self.cfg_is_masked_until is not None:
                until = (C.c_int64 * len(self.cfg_is_masked_until))(*[int(v) for v in self.cfg_is_masked_until])
            _lib.check(self._lib.b200_lm_set_cfg(self._h, float(self.cfg_coef), int(bool(self.cfg_is_no_text)), until,
                                                 0 if until is None else len(self.cfg_is_masked_until)))
            if lm.cfg.cross_attention:       # the condition memory holds T keys per row for the whole session
                _lib.check(self._lib.b200_lm_set_cross_len(self._h, int(condition_cross.shape[1])))
            self._stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.b200_lm_streaming_begin(self._h, int(batch_size), C.c_void_p(self._stream)))
            # one draw from torch's CPU generator seeds the session's in-step noise stream
            seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
            _lib.check(self._lib.b200_lm_seed_noise(self._h, C.c_uint64(seed)))
            if condition_sum is not None:
                cs = condition_sum.reshape(model_batch, lm.dim).contiguous()
                _lib.check(self._lib.b200_lm_set_condition_sum(self._h, _lib.ptr(cs), model_batch))
        self._batch = int(batch_size)
        self._model_batch = model_batch
        if condition_cross is not None:
            self.set_condition_cross(condition_cross)
        self._noise_per_row = int(self._lib.b200_lm_noise_per_row(self._h))
        self._kt = min(self.top_k_text, lm.text_card)
        self._ka = min(self.top_k, lm.card)
        self._streaming_state = self

    def _stop(self) -> None:
        if self._batch is not None:
            with self._device():
                self._lib.b200_lm_streaming_end(self._h)
            self._batch = None
            self._streaming_state = None

    def streaming(self, batch_size: int) -> ExitStack:
        stack = ExitStack()
        self._start(batch_size)
        stack.callback(self._stop)
        return stack

    def streaming_forever(self, batch_size: int) -> None:
        self._start(batch_size)

    def _mask(self, mask: torch.Tensor) -> torch.Tensor:
        mask = mask.to(device=self.lm_model.device, dtype=torch.bool).contiguous()
        assert mask.shape == (self._batch,)
        return mask

    def reset_streaming(self, reset_mask: torch.Tensor | None = None) -> None:
        assert self._batch is not None, "Trying to reset streaming, but lm_gen wasn't streaming."
        m = None if reset_mask is None else self._mask(reset_mask)
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_reset(self._h, _lib.ptr(m)))

    def set_condition_cross(self, cross: torch.Tensor, rows: tp.Sequence[int] | torch.Tensor | None = None) -> None:
        """Replaces the condition memory (``_MHAState.k_cross / v_cross`` of every cross-attention layer) of model rows ``rows``
        (None: all of them) with the keys and values of ``cross`` [len(rows), T, dim], e.g. ``fuser.get_cross`` of new condition
        tensors: what the TTS service does when a slot takes a new voice (tts.py:422-440).  Model rows are the sessions ``b``
        and, under classifier-free guidance, ``batch + b`` for their null half.  T is the one the session started with.  The
        rows' positions and every other row are unchanged; ``reset_streaming`` keeps the memory, as in the reference."""
        assert self._batch is not None, "lm_gen is not streaming"
        assert self.lm_model.cfg.cross_attention, "the model has no cross-attention layers"
        if rows is not None:
            rows = [int(r) for r in (rows.tolist() if isinstance(rows, torch.Tensor) else rows)]
        n = self._model_batch if rows is None else len(rows)
        src = cross.to(device=self.lm_model.device, dtype=self.lm_model.dtype).contiguous()
        assert src.dim() == 3 and src.shape[0] == n and src.shape[2] == self.lm_model.dim, \
            f"expected a condition [{n}, T, {self.lm_model.dim}], got {tuple(src.shape)}"
        keys = self._entry_shape("layers.0.k_cross")[2]
        assert src.shape[1] == keys, f"the condition memory holds {keys} keys per row for this session, got {src.shape[1]}"
        rows_c = None if rows is None else (C.c_int32 * n)(*rows)
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_set_condition_cross(self._h, _lib.ptr(src), rows_c, n))

    _ROW_SAMPLING = ("temp_text", "temp", "top_k_text", "top_k", "pad_mult", "repetition_context", "repetition_penalty")

    def set_session_sampling(self, rows: tp.Sequence[int] | torch.Tensor, temp_text: float | None = None, temp: float | None = None,
                             top_k_text: int | None = None, top_k: int | None = None, pad_mult: float | None = None,
                             repetition_context: int | None = None, repetition_penalty: float | None = None) -> None:
        """Gives sessions ``rows`` their own sampling settings (``session_sampling`` must be set before streaming).  A setting
        left at None takes the handle-wide value (``temp_text``, ``temp``, ``top_k_text``, ``top_k`` of this LMGen; pad_mult 0,
        repetition_context 0, repetition_penalty 1); all of them None returns the rows to the handle-wide values, which they then
        follow as they change.  Text tokens: the rows' recent text (the newest ``repetition_context`` tokens of their history,
        padding and initial tokens left out) is penalised, l / penalty where l >= 0 and l * penalty below, then a sampling row
        samples at ``temp_text`` with ``pad_mult`` added to the padding token's tempered score, over its ``top_k_text``; a
        greedy row takes the argmax of the penalised logits.  Audio tokens use ``temp`` and ``top_k``.  Top-k values must lie in
        [1, this LMGen's]; ValueError outside the ranges, and nothing changes.  Ordered before the next step."""
        assert self._batch is not None, "lm_gen is not streaming"
        if not self.session_sampling:
            raise RuntimeError("per-session sampling is off: set lm_gen.session_sampling before streaming")
        rows = [int(r) for r in (rows.tolist() if isinstance(rows, torch.Tensor) else rows)]
        for r in rows:
            if not 0 <= r < self._batch:
                raise ValueError(f"row {r} outside [0, {self._batch})")
        vals = dict(temp_text=temp_text, temp=temp, top_k_text=top_k_text, top_k=top_k, pad_mult=pad_mult,
                    repetition_context=repetition_context, repetition_penalty=repetition_penalty)
        p = None
        if any(v is not None for v in vals.values()):
            for k in ("top_k_text", "top_k", "repetition_context"):
                if vals[k] is not None and (isinstance(vals[k], bool) or int(vals[k]) != vals[k]):
                    raise ValueError(f"{k} must be an integer, got {vals[k]!r}")
            base = dict(temp_text=self.temp_text, temp=self.temp, top_k_text=self.top_k_text, top_k=self.top_k, pad_mult=0.0,
                        repetition_context=0, repetition_penalty=1.0)
            one = _lib.RowSamplingC(**{k: (base[k] if vals[k] is None else vals[k]) for k in self._ROW_SAMPLING})
            p = (_lib.RowSamplingC * max(len(rows), 1))(*([one] * len(rows)))
        rows_c = (C.c_int32 * max(len(rows), 1))(*rows)
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_set_row_sampling(self._h, rows_c, len(rows), p))

    def _entry_shape(self, name: str) -> tuple[int, ...]:
        for n, _, shape, _ in self._state_entries():
            if n == name:
                return shape
        raise KeyError(name)

    def set_exec_mask(self, exec_mask: torch.Tensor) -> None:
        assert self._batch is not None
        m = self._mask(exec_mask)
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_set_exec_mask(self._h, _lib.ptr(m)))

    # ---- streaming state ------------------------------------------------------------------------------
    def _state_entries(self) -> list[tuple[str, torch.dtype, tuple[int, ...], int]]:
        out = []
        for i in range(int(self._lib.b200_lm_state_count(self._h))):
            name, dt, nd, nb = C.c_char_p(), C.c_int(), C.c_int(), C.c_int64()
            shape = (C.c_int64 * 8)()
            _lib.check(self._lib.b200_lm_state_entry(self._h, i, C.byref(name), C.byref(dt), C.byref(nd), shape, C.byref(nb)))
            out.append((name.value.decode(), _TORCH_DTYPES[dt.value], tuple(shape[:nd.value]), nb.value))
        return out

    def _read_state(self, name: str, dtype: torch.dtype, shape: tuple[int, ...], nbytes: int) -> torch.Tensor:
        t = torch.empty(shape, dtype=dtype, device=self.lm_model.device)
        _lib.check(self._lib.b200_lm_state_read(self._h, name.encode(), _lib.ptr(t), nbytes))
        return t

    def _write_state(self, name: str, t: torch.Tensor) -> None:
        t = t.to(self.lm_model.device).contiguous()
        _lib.check(self._lib.b200_lm_state_write(self._h, name.encode(), _lib.ptr(t), t.numel() * t.element_size()))

    def get_streaming_state(self) -> dict[str, tp.Any]:
        """``StreamingModule.get_streaming_state`` (streaming.py:158-166): module path -> state, with the reference's field
        names (``_LMGenState`` lm.py:523-535 under ``""``; the temporal transformer's ``_MHAState`` / ``RingKVCache``
        transformer.py:196-288, 321-334 under ``lm_model.transformer.layers.<i>.self_attn``; the reference keeps the model's
        states behind ``set_streaming_detached``, here they are part of the snapshot so that it can be restored).  The
        tensors are copies."""
        assert self._batch is not None, "lm_gen is not streaming"
        with self._device():
            self._sync_stream()
            raw = {name: self._read_state(name, dt, shape, nb) for name, dt, shape, nb in self._state_entries()}
            offset_cpu = int(self._lib.b200_lm_get_offset_cpu(self._h))
        state: dict[str, tp.Any] = {}
        state[""] = SimpleNamespace(batch_size=self._batch, device=self.lm_model.device, cache=raw["cache"], offsets=raw["offsets"],
                                    offset_cpu=offset_cpu, exec_mask=raw["exec_mask"].bool(),
                                    noise_counter=raw["noise_counter"])
        if "session_sampling.params" in raw:          # per-session settings [B, 8], text histories [B, N] and their counts [B]
            state[""].session_sampling = SimpleNamespace(params=raw["session_sampling.params"], history=raw["session_sampling.history"],
                                                         count=raw["session_sampling.count"])
        mexec = raw.get("model.exec_mask", raw["exec_mask"]).bool()
        state["lm_model"] = SimpleNamespace(batch_size=self._model_batch, exec_mask=mexec)
        state["lm_model.transformer"] = SimpleNamespace(batch_size=self._model_batch, exec_mask=mexec, offsets=raw["model.offset"])
        for i in range(self.lm_model.cfg.num_layers):
            p = f"layers.{i}"
            if p + ".k" in raw:
                kv = SimpleNamespace(cache=torch.stack([raw[p + ".k"], raw[p + ".v"]]), end_offset=raw["model.offset"].clone())
            else:
                kv = SimpleNamespace(cache_q8=torch.stack([raw[p + ".k8"], raw[p + ".v8"]]),
                                     scales=torch.stack([raw[p + ".k_scale"], raw[p + ".v_scale"]]),
                                     end_offset=raw["model.offset"].clone())
            state[f"lm_model.transformer.layers.{i}.self_attn"] = SimpleNamespace(
                batch_size=self._model_batch, exec_mask=mexec, kv_cache=kv, offset=raw["model.offset"].clone(), offset_cpu=offset_cpu)
            if p + ".k_cross" in raw:     # _MHAState of the cross-attention module (transformer.py:321-327): only its memory
                state[f"lm_model.transformer.layers.{i}.cross_attention"] = SimpleNamespace(
                    batch_size=self._model_batch, exec_mask=mexec, kv_cache=None, k_cross=raw[p + ".k_cross"],
                    v_cross=raw[p + ".v_cross"])
        return state

    def set_streaming_state(self, state: dict[str, tp.Any]) -> None:
        """``set_streaming_state`` (streaming.py:168-181): every module state must be present and nothing else."""
        assert self._batch is not None, "lm_gen is not streaming"
        state = dict(state)
        L = self.lm_model.cfg.num_layers
        expected = ["", "lm_model", "lm_model.transformer"] + [f"lm_model.transformer.layers.{i}.self_attn" for i in range(L)]
        if self.lm_model.cfg.cross_attention:
            expected += [f"lm_model.transformer.layers.{i}.cross_attention" for i in range(L)]
        for name in expected:
            if name not in state:
                raise RuntimeError(f"Expected to find a streaming state for {name}.")
        root = state.pop("")
        assert root.batch_size == self._batch, "snapshot was taken with another batch size"
        with self._device():
            self._sync_stream()
            self._write_state("cache", root.cache.long())
            self._write_state("offsets", root.offsets.long())
            self._write_state("exec_mask", root.exec_mask.to(torch.uint8))
            if hasattr(root, "noise_counter"):
                self._write_state("noise_counter", root.noise_counter.long())
            if self.session_sampling:
                ss = root.session_sampling
                self._write_state("session_sampling.params", ss.params.float())
                self._write_state("session_sampling.history", ss.history.int())
                self._write_state("session_sampling.count", ss.count.int())
            _lib.check(self._lib.b200_lm_set_offset_cpu(self._h, int(root.offset_cpu)))
            tr = state.pop("lm_model.transformer")
            state.pop("lm_model")
            self._write_state("model.offset", tr.offsets.long())
            if self.cfg_coef != 1.:
                self._write_state("model.exec_mask", tr.exec_mask.to(torch.uint8))
            for i in range(L):
                st = state.pop(f"lm_model.transformer.layers.{i}.self_attn")
                kv = st.kv_cache
                if hasattr(kv, "cache"):
                    self._write_state(f"layers.{i}.k", kv.cache[0])
                    self._write_state(f"layers.{i}.v", kv.cache[1])
                else:
                    self._write_state(f"layers.{i}.k8", kv.cache_q8[0])
                    self._write_state(f"layers.{i}.v8", kv.cache_q8[1])
                    self._write_state(f"layers.{i}.k_scale", kv.scales[0])
                    self._write_state(f"layers.{i}.v_scale", kv.scales[1])
                if self.lm_model.cfg.cross_attention:
                    cx = state.pop(f"lm_model.transformer.layers.{i}.cross_attention")
                    self._write_state(f"layers.{i}.k_cross", cx.k_cross)
                    self._write_state(f"layers.{i}.v_cross", cx.v_cross)
        if state:
            raise RuntimeError(f"Some states were not consumed: {list(state.keys())}")

    # ---- one session -----------------------------------------------------------------------------
    def export_session(self, row: int) -> torch.Tensor:
        """Session ``row`` as a uint8 record on the model's device (``b200_lm_session_export``): its token ring, offsets,
        positions and the temporal K/V of its live fill, so the size follows the fill, and on a cross-attention model its
        condition memory.  The row is not changed and keeps
        running; reset it once the session has moved.  A short-ring row past ``kv_capacity`` raises (its history is lost)."""
        assert self._batch is not None, "lm_gen is not streaming"
        n = C.c_int64()
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_session_bytes(self._h, int(row), C.byref(n)))
            rec = torch.empty(n.value, dtype=torch.uint8, device=self.lm_model.device)
            _lib.check(self._lib.b200_lm_session_export(self._h, int(row), _lib.ptr(rec), n.value))
        return rec

    def import_session(self, row: int, record: torch.Tensor) -> None:
        """Replaces session ``row`` with a record of ``export_session`` from any handle of the same model configuration and
        KV storage type, on any device (``.to(device)`` copies it across GPUs).  Nothing changes if it is refused: ValueError
        for an incompatible record or row, ``B200Error`` when the ring or the pool cannot hold the session's history."""
        assert self._batch is not None, "lm_gen is not streaming"
        rec = record.to(self.lm_model.device).contiguous()
        assert rec.dtype == torch.uint8 and rec.dim() == 1, "a session record is a 1-d uint8 tensor"
        with self._device():
            self._sync_stream()
            _lib.check(self._lib.b200_lm_session_import(self._h, int(row), _lib.ptr(rec), rec.numel()))

    # ---- sampling noise --------------------------------------------------------------------------
    def draw_noise(self) -> torch.Tensor | None:
        """Exp(1) draws of one step in the reference's order (lm.py:736 then lm.py:836 x dep_q), each
        ``torch.empty(B, k).exponential_(1)`` on the model device, packed as [B, kt + dep_q*ka].  Not used by ``step`` itself
        (which draws inside the library); for callers that want torch's generator to own the stream."""
        if not (self.use_sampling and (self.temp > 0 or self.temp_text > 0)):
            return None
        B, dev = self._batch, self.lm_model.device
        parts = [torch.empty(B, self._kt, device=dev, dtype=torch.float32).exponential_(1)]
        for _ in range(self.lm_model.dep_q):
            parts.append(torch.empty(B, self._ka, device=dev, dtype=torch.float32).exponential_(1))
        return torch.cat(parts, dim=1).contiguous()

    def pack_noise(self, noise_text: torch.Tensor, noise_audio: tp.Sequence[torch.Tensor]) -> torch.Tensor:
        dev = self.lm_model.device
        return torch.cat([noise_text.to(dev)] + [n.to(dev) for n in noise_audio], dim=1).float().contiguous()

    def read_buffer(self, name: str, dtype: torch.dtype, shape: tuple[int, ...]) -> torch.Tensor:
        out = torch.empty(shape, device=self.lm_model.device, dtype=dtype)
        n = C.c_int64()
        with self._device():
            _lib.check(self._lib.b200_lm_read_buffer(self._h, name.encode(), _lib.ptr(out),
                                                     out.numel() * out.element_size(), C.byref(n)))
        assert n.value == out.numel() * out.element_size(), (name, n.value, shape)
        return out

    def error_flags(self) -> int:
        """Synchronises and returns (and clears) the device error flags (1 = a token id outside its embedding table, 4 = a session
        stepped past a shortened KV ring, `kv_capacity`; 8 = a session's KV ring did not get a page because the `kv_pool_frames`
        pool was full: that session's output is garbage until it is reset, the others are unaffected)."""
        v = C.c_int(0)
        with self._device():
            _lib.check(self._lib.b200_lm_error_flags(self._h, C.byref(v)))
        return v.value

    def kv_pool_usage(self) -> tuple[int, int]:
        """(pages held by the model's rows, pages in the pool) of a `kv_pool_frames` handle; (0, 0) without a pool.  Synchronises."""
        used, total = C.c_int(0), C.c_int(0)
        with self._device():
            _lib.check(self._lib.b200_lm_kv_pool_usage(self._h, C.byref(used), C.byref(total)))
        return used.value, total.value

    # ---- the step ---------------------------------------------------------------------------------
    @torch.no_grad()
    def _step(self, input_tokens: torch.Tensor, depformer_replace_tokens=None, noise: torch.Tensor | None = None):
        if self._batch is None:
            raise RuntimeError("You should wrap those calls with a `with lm_gen.streaming(): ...`.")   # lm.py:673-676
        lm = self.lm_model
        assert input_tokens.dim() == 3, "Shape should be [B, K, T]."
        B, Ki, S = input_tokens.shape
        assert B == self._batch, f"Got a batch size {B}, expected {self._batch}"
        assert S == 1, "Only support being given steps one by one."
        needed = lm.num_codebooks - lm.dep_q - 1
        assert Ki >= needed, f"We expect {needed} tokens from the user stream, got {Ki}."
        codes = input_tokens[:, :needed, 0].to(device=lm.device, dtype=torch.int64).contiguous()
        if noise is not None:
            noise = noise.to(device=lm.device, dtype=torch.float32).contiguous()
            assert noise.shape == (B, self._noise_per_row), f"noise must be [{B}, {self._noise_per_row}]"
        out = torch.empty(B, lm.dep_q + 1, device=lm.device, dtype=torch.int64)
        ready = C.c_int(0)
        replace = None
        if depformer_replace_tokens is not None:            # lm.py:751-755
            assert depformer_replace_tokens.dim() == 3
            replace = depformer_replace_tokens.squeeze(-1).to(device=lm.device, dtype=torch.int64).contiguous()
            assert replace.shape == (B, lm.dep_q), f"expected [{B}, {lm.dep_q}, 1] replacement tokens"
        with self._device():
            self._push_sampling()
            self._sync_stream()
            _lib.check(self._lib.b200_lm_step_ex(self._h, _lib.ptr(codes), needed, _lib.ptr(noise), _lib.ptr(replace), _lib.ptr(out),
                                                 int(self.support_out_of_sync), C.byref(ready)))
        if self.check:                                      # lm.py:704-711: no ungenerated / out-of-range token may reach the model
            assert self.error_flags() == 0, "a token outside its embedding table reached the model"
        if self.on_text_logits_hook is not None:
            tl = self.read_buffer("text_logits", torch.bfloat16, (B, lm.text_card))
            self.on_text_logits_hook(tl[:, None, None, :])
        if self.on_text_hook is not None:
            self.on_text_hook(self.read_buffer("text_token", torch.int64, (B,)))
        if self.on_audio_hook is not None and lm.dep_q > 0:
            self.on_audio_hook(self.read_buffer("audio_tokens", torch.int64, (lm.dep_q, B)).t().contiguous())
        if not ready.value:
            return None
        return out[:, :, None]

    def step(self, input_tokens: torch.Tensor, depformer_replace_tokens=None,
             noise: torch.Tensor | None = None) -> torch.Tensor | None:
        return self._step(input_tokens, depformer_replace_tokens, noise)

    def step_with_extra_heads(self, input_tokens: torch.Tensor, depformer_replace_tokens=None,
                              noise: torch.Tensor | None = None):
        """lm.py:793-807: ``(tokens, [softmax(extra_head(transformer_out)) ...])``, each head ``[B, 1, extra_heads_dim]``."""
        out = self._step(input_tokens, depformer_replace_tokens, noise)
        if out is None:
            return None
        cfg = self.lm_model.cfg
        n, E, MB = cfg.extra_heads_num_heads, cfg.extra_heads_dim, self._model_batch
        if n == 0:
            return out, []
        heads = self.read_buffer("extra_heads", torch.bfloat16, (n, MB, E))
        return out, [heads[i][:, None, :] for i in range(n)]

    def step_host(self, codes_cpu: torch.Tensor, noise_cpu: torch.Tensor | None, out_cpu: torch.Tensor) -> bool:
        """Host-buffer step (H2D of codes/noise and D2H of tokens inside): i64 [B, n_in] -> i64 [B, dep_q+1]."""
        ready = C.c_int(0)
        with self._device():
            self._push_sampling()
            self._sync_stream()
            _lib.check(self._lib.b200_lm_step_host(self._h, _lib.ptr(codes_cpu), codes_cpu.shape[1], _lib.ptr(noise_cpu),
                                                   _lib.ptr(out_cpu), int(self.support_out_of_sync), C.byref(ready)))
        return bool(ready.value)

    def assume_fill(self, fill: int) -> None:
        with self._device():
            _lib.check(self._lib.b200_lm_assume_fill(self._h, int(fill)))

    def algorithmic_bytes(self, kv_fill: int) -> int:
        return int(self._lib.b200_lm_algorithmic_bytes(self._h, int(kv_fill)))
