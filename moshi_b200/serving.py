"""Session placement for multi-GPU serving: replicas only.

Dialogue sessions are independent (every state tensor is ``[B, ...]`` and every reduction is per
row), so N GPUs run N replicas of the weights, each owning a contiguous shard of the session slots;
there is no data-path collective (SURVEY.md 8e; the reference deploys one process per GPU behind a
load balancer, ``swarm-config.yml:48-63``).  ``torch.distributed`` is used only to launch one
process per GPU and to reduce timings / counts in the benchmark.
"""
from __future__ import annotations

import os
import typing as tp

import torch


def shard_sessions(total: int, world_size: int, rank: int) -> range:
    """Contiguous, balanced shard of session slots [0, total) for ``rank``."""
    base, extra = divmod(total, world_size)
    start = rank * base + min(rank, extra)
    return range(start, start + base + (1 if rank < extra else 0))


def init_distributed(backend: str | None = None) -> tuple[int, int]:
    """(rank, world_size) from the torchrun environment; initialises the process group if world > 1."""
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group(backend=backend)
    return rank, world


def _reduce(value: float, op) -> float:
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return value
    dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
    t = torch.tensor([value], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=op)
    return float(t.item())


def max_over_ranks(value: float) -> float:
    import torch.distributed as dist
    return _reduce(value, dist.ReduceOp.MAX)


def sum_over_ranks(value: float) -> float:
    import torch.distributed as dist
    return _reduce(value, dist.ReduceOp.SUM)


def barrier() -> None:
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.barrier()


# ---------------------------------------------------------------------------------------------------
# One frame for every session slot of this GPU (SURVEY.md 8f item 1: the caller's per-frame plumbing)
# ---------------------------------------------------------------------------------------------------
NODATA, ACTIVE, RESET = 0, -1, -2      # UpdateFlags of rust/moshi-server/batched_asr.py:23-30


class SessionRecord(tp.NamedTuple):
    """One dialogue session of a ``DialogueService``: its LM and Mimi records (uint8 device tensors)."""
    lm: torch.Tensor
    mimi: torch.Tensor


class DialogueService:
    """Batched full-duplex frame step with the calling convention of ``ASRService.step``
    (``rust/moshi-server/batched_asr.py:100-215``, bound by ``py_basr_module.rs``): numpy host buffers in and
    out, per-slot update flags, state owned by the service.  The body of the reference's loop
    (``server.py:120-147``: ``mimi.encode -> lm_gen.step -> mimi.decode -> .cpu()``) runs below the C ABI as one
    stream-ordered chain with a single host wait (``b200_frame_step``); masks and the "row is past its delay
    warm-up" decision are built on the device.
    """

    def __init__(self, batch_size: int, lm, mimi, use_sampling: bool = True, temp: float = 0.8, temp_text: float = 0.7,
                 top_k: int = 250, top_k_text: int = 25, kv_dtype: str = "bf16", kv_capacity: int | None = None,
                 kv_pool_frames: int | None = None, session_sampling: int | None = None):
        import ctypes as C

        from . import _lib
        from .models import LMGen
        self.batch_size = batch_size
        # the handle-wide values a session's missing settings take (protocol.FrontEnd.connect)
        self.sampling_defaults = dict(temp_text=temp_text, temp=temp, top_k_text=top_k_text, top_k=top_k)
        self.session_sampling = session_sampling    # tokens of text history per session, or None: no per-session settings
        self.lm, self.mimi = lm, mimi
        self.lm_gen = LMGen(lm, use_sampling=use_sampling, temp=temp, temp_text=temp_text, top_k=top_k, top_k_text=top_k_text,
                            support_out_of_sync=True)
        self.lm_gen.kv_dtype = kv_dtype
        self.lm_gen.kv_capacity = kv_capacity
        self.lm_gen.kv_pool_frames = kv_pool_frames
        self.lm_gen.session_sampling = session_sampling
        self.lm_gen.streaming_forever(batch_size)
        self.mimi.streaming_forever(batch_size)
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._lib.b200_frame_create(mimi._h, lm._h, batch_size, mimi.num_codebooks, lm.dep_q, mimi.frame_size,
                                               _lib.current_stream(lm.device), C.byref(self._h)))
        self.frame_size = mimi.frame_size
        self.tokens_per_slot = lm.dep_q + 1

    def read_buffer(self, name: str, dtype: torch.dtype, shape: tuple) -> torch.Tensor:
        """Hand-off of the last frame (``b200_frame_read_buffer``): "codes_in", "tokens", "codes_out", "exec", "decoder_exec"."""
        import ctypes as C

        from . import _lib
        out = torch.empty(shape, dtype=dtype, device=self.lm.device)
        n = C.c_int64()
        _lib.check(self._lib.b200_frame_read_buffer(self._h, name.encode(), _lib.ptr(out), out.numel() * out.element_size(), C.byref(n)))
        assert n.value == out.numel() * out.element_size(), (name, n.value, shape)
        return out

    def release(self, slots) -> None:
        """Resets the LM and Mimi rows of closed session slots, so that a paged LM (``kv_pool_frames``) returns their KV pages to
        the pool now rather than when the slot's next session sends its RESET frame."""
        mask = torch.zeros(self.batch_size, dtype=torch.bool)
        mask[list(slots)] = True
        if mask.any():
            self.lm_gen.reset_streaming(mask)
            self.mimi.reset_streaming(mask)

    def set_session_sampling(self, slot: int, **settings) -> None:
        """Session ``slot``'s own sampling settings (``LMGen.set_session_sampling``; the service was built with
        ``session_sampling``); none given returns it to the service-wide values.  They apply from the next ``step`` on and
        stay across that slot's RESET frames until they are set again."""
        self.lm_gen.set_session_sampling([slot], **settings)

    def export_session(self, slot: int) -> "SessionRecord":
        """The LM and Mimi state of session ``slot`` as device records (``LMGen.export_session``, ``MimiModel.export_session``).
        The slot is not changed; once the session has moved, call ``release([slot])`` so that a paged LM gets its pages back."""
        return SessionRecord(self.lm_gen.export_session(slot), self.mimi.export_session(slot))

    def import_session(self, slot: int, record: "SessionRecord") -> None:
        """Continues a session exported from another service (same models, KV storage type; any GPU) in ``slot``.  The next
        ``step``'s update for the slot must be ``ACTIVE``: ``RESET`` would erase the imported session.  The source calls
        ``release([slot])`` on its own slot to return its pages.  PCM still buffered in a ``SessionPool`` is the caller's to carry.
        The LM record is checked and imported first: if it is refused, nothing changes."""
        self.lm_gen.import_session(slot, record.lm)
        self.mimi.import_session(slot, record.mimi)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.b200_frame_destroy(self._h)
            self._h = None
            self.lm_gen._stop()
            self.mimi._stop()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _np_ptr(a, dtype, numel: int, name: str):
        import ctypes as C

        import numpy as np
        if a is None:
            return C.c_void_p(0)
        if not isinstance(a, np.ndarray) or a.dtype != dtype or not a.flags["C_CONTIGUOUS"] or a.size != numel:
            raise AssertionError(f"{name}: expected a C-contiguous {np.dtype(dtype).name} array of {numel} elements")
        return C.c_void_p(a.ctypes.data)

    def step(self, batch_pcm, pcm_out, tokens_out, updates=None, flags_out=None, noise=None) -> None:
        """``batch_pcm`` f32 [B * frame_size] (as the Rust harness passes it, ``batched_asr.py:193-196``) -> ``pcm_out``
        f32 [B, frame_size], ``tokens_out`` i64 [B, dep_q + 1], ``flags_out`` u8 [B] (1 = the slot produced a frame).
        ``updates``: per-slot NODATA / ACTIVE / RESET (or a positive marker), None = unchanged.
        ``noise``: f32 [B, noise_per_row] Exp(1) draws (numpy or CUDA tensor); None = drawn on the device."""
        import ctypes as C

        import numpy as np

        from . import _lib
        B = self.batch_size
        upd = None
        if updates is not None:
            upd = np.ascontiguousarray(np.asarray(updates, dtype=np.int32))
            assert upd.shape == (B,), f"expected {B} slot updates"
        noise_host = noise_dev = C.c_void_p(0)
        keep = None
        if noise is None:
            pass                      # both NULL: the LM step draws its Exp(1) noise itself, inside its CUDA graph
        elif isinstance(noise, np.ndarray):
            noise_host = self._np_ptr(noise, np.float32, B * self._lib.b200_lm_noise_per_row(self.lm._h), "noise")
        else:
            keep = noise.to(device=self.lm.device, dtype=torch.float32).contiguous()
            noise_dev = _lib.ptr(keep)
        _lib.check(self._lib.b200_frame_step(
            self._h, self._np_ptr(batch_pcm, np.float32, B * self.frame_size, "batch_pcm"),
            self._np_ptr(upd, np.int32, B, "updates"), noise_host, noise_dev,
            self._np_ptr(pcm_out, np.float32, B * self.frame_size, "pcm_out"),
            self._np_ptr(tokens_out, np.int64, B * self.tokens_per_slot, "tokens_out"),
            self._np_ptr(flags_out, np.uint8, B, "flags_out")))


MASK_ACTIVE, MASK_MARKER_RECEIVED, MASK_IS_EOS = 1, 2, 4     # MaskFlags of rust/moshi-server/batched_asr.py:14-20


class ASRService:
    """``ASRService`` of ``rust/moshi-server/batched_asr.py:100-213`` for the speech-to-text models (``dep_q = 0``, extra heads),
    with its calling convention: ``step(batch_pcm, flags_out, tokens_out, extra_heads, updates)`` every 80 ms for all slots,
    numpy buffers in and out, as ``py_basr_module.rs`` calls it.  The per-slot client state (``ClientState``, :85-98) and the
    end-of-stream countdown live on the device; a frame (updates -> resets -> ``mimi.encode`` -> ``step_with_extra_heads`` ->
    flags) is one stream-ordered chain with a single host wait (``b200_asr_step``).  Construction runs the reference's warm-up
    (:119-130); afterwards every slot is inactive until its first ``ACTIVE`` or ``RESET``."""

    def __init__(self, batch_size: int, lm, mimi, asr_delay_in_tokens: int = 32, temp: float = 0.0, kv_dtype: str = "bf16",
                 kv_capacity: int | None = None, kv_pool_frames: int | None = None):
        import ctypes as C

        import numpy as np

        from . import _lib
        from .models import LMGen
        self.batch_size = batch_size
        self.lm, self.mimi = lm, mimi
        self.asr_delay_in_tokens = asr_delay_in_tokens
        self.lm_gen = LMGen(lm, temp_text=temp)                     # batched_asr.py:114
        self.lm_gen.kv_dtype = kv_dtype
        self.lm_gen.kv_capacity = kv_capacity
        self.lm_gen.kv_pool_frames = kv_pool_frames
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        self.lm_gen.streaming_forever(batch_size)
        try:
            self.mimi.streaming_forever(batch_size)
        except BaseException:
            self.lm_gen._stop()
            raise
        try:
            with torch.cuda.device(lm.device):
                _lib.check(self._lib.b200_asr_create(mimi._h, lm._h, batch_size, int(asr_delay_in_tokens),
                                                     _lib.current_stream(lm.device), C.byref(self._h)))
        except BaseException:
            self._h = None
            self.lm_gen._stop()
            self.mimi._stop()
            raise
        self.frame_size = mimi.frame_size
        self.extra_heads_num_heads = lm.cfg.extra_heads_num_heads
        self._tokens = np.zeros(batch_size, dtype=np.int64)

    def read_buffer(self, name: str, dtype: torch.dtype, shape: tuple) -> torch.Tensor:
        """Buffers of the last frame (``b200_asr_read_buffer``): "codes_in", "tokens", "extra_heads", "exec", "reset", "offset",
        "real_end"."""
        import ctypes as C

        from . import _lib
        out = torch.empty(shape, dtype=dtype, device=self.lm.device)
        n = C.c_int64()
        _lib.check(self._lib.b200_asr_read_buffer(self._h, name.encode(), _lib.ptr(out), out.numel() * out.element_size(), C.byref(n)))
        assert n.value == out.numel() * out.element_size(), (name, n.value, shape)
        return out

    def release(self, slots) -> None:
        """Resets the LM and Mimi rows of closed session slots, so that a paged LM (``kv_pool_frames``) returns their KV pages to
        the pool now.  The slot's client state is left as it is: its next session still starts with ``RESET``."""
        mask = torch.zeros(self.batch_size, dtype=torch.bool)
        mask[list(slots)] = True
        if mask.any():
            self.lm_gen.reset_streaming(mask)
            self.mimi.reset_streaming(mask)

    def export_session(self, slot: int) -> SessionRecord:
        """The LM and Mimi state of session ``slot`` as device records (see ``DialogueService.export_session``).  The client
        state (offset, end-of-stream countdown) does not travel: move a session before it sends its end-of-stream marker."""
        return SessionRecord(self.lm_gen.export_session(slot), self.mimi.export_session(slot))

    def import_session(self, slot: int, record: SessionRecord) -> None:
        """Continues a session exported from another service in ``slot``; its next update must be ``ACTIVE`` (``RESET`` would
        erase it).  The LM record is checked and imported first: if it is refused, nothing changes."""
        self.lm_gen.import_session(slot, record.lm)
        self.mimi.import_session(slot, record.mimi)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.b200_asr_destroy(self._h)
            self._h = None
            self.lm_gen._stop()
            self.mimi._stop()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def step(self, batch_pcm, flags_out, tokens_out, extra_heads, updates) -> bool:
        """``ASRService.step`` (batched_asr.py:132-213).  ``batch_pcm`` f32 [B * frame_size]; ``flags_out`` u8 [B], read and
        written (entries the reference does not assign keep their value); ``tokens_out`` any integer dtype [B], assigned like the
        reference (``tokens_out[:] = ...``: -2 wraps in an unsigned array); ``extra_heads`` f32 [B, extra_heads_num_heads];
        ``updates`` B ints (NODATA / ACTIVE / RESET, or a positive end-of-stream marker).  Returns whether the model ran: when
        no slot is active, tokens and extra heads are not written."""
        import ctypes as C

        import numpy as np

        from . import _lib
        B, n = self.batch_size, self.extra_heads_num_heads
        upd = np.ascontiguousarray(np.asarray(updates, dtype=np.int32))
        assert upd.shape == (B,), f"expected {B} slot updates"
        assert isinstance(tokens_out, np.ndarray) and tokens_out.shape == (B,) and np.issubdtype(tokens_out.dtype, np.integer), \
            f"tokens_out: expected an integer array of shape ({B},)"
        assert isinstance(extra_heads, np.ndarray) and extra_heads.shape == (B, n), f"extra_heads: expected shape ({B}, {n})"
        ran = C.c_int(0)
        _np = DialogueService._np_ptr
        with torch.cuda.device(self.lm.device):
            _lib.check(self._lib.b200_asr_step(
                self._h, _np(batch_pcm, np.float32, B * self.frame_size, "batch_pcm"), _np(upd, np.int32, B, "updates"),
                _np(flags_out, np.uint8, B, "flags_out"), _np(self._tokens, np.int64, B, "tokens"),
                _np(extra_heads, np.float32, B * n, "extra_heads") if n else C.c_void_p(0), C.byref(ran)))
        if ran.value:
            tokens_out[:] = self._tokens
        return bool(ran.value)


class SessionPool:
    """Slot allocator and PCM framing in front of ``DialogueService.step`` (host logic only; no device work).

    The reference's single-session server accumulates decoded opus PCM in ``all_pcm_data`` and cuts 1920-sample frames off
    its front (``server.py:116-126``); the batched Rust server keeps one such buffer per slot and tells the Python side every
    80 ms which slots are ``ACTIVE`` / ``RESET`` / have ``NODATA`` (``batched_asr.py:23-30,146-170``).  This class is that
    bookkeeping for ``batch_size`` slots:

    * ``open()`` hands out a free slot (the first frame it contributes carries ``RESET``), ``close(slot)`` returns it;
    * ``push_pcm(slot, samples)`` appends any number of float32 samples to the slot's buffer;
    * ``next_frame(batch_pcm, updates)`` fills one frame per slot that has >= ``frame_size`` samples buffered (``ACTIVE``, or
      ``RESET`` for a slot's first frame) and marks the others ``NODATA`` — exactly the arrays ``DialogueService.step`` takes;
      it returns the slots that contributed a frame;
    * sessions are independent, so a slot that falls behind simply skips frames (``NODATA``) without stalling the batch.
    """

    def __init__(self, batch_size: int, frame_size: int = 1920, max_buffered_frames: int = 50):
        import numpy as np
        self.batch_size, self.frame_size = batch_size, frame_size
        self.max_samples = max_buffered_frames * frame_size
        self._free = list(range(batch_size - 1, -1, -1))            # pop() hands out slot 0 first
        self._open: dict[int, bool] = {}                            # slot -> still needs its RESET frame
        self._buf = [np.zeros(0, dtype=np.float32) for _ in range(batch_size)]
        self.frames_in = [0] * batch_size

    @property
    def free_slots(self) -> int:
        return len(self._free)

    def open(self) -> int:
        if not self._free:
            raise RuntimeError("no free session slot")
        slot = self._free.pop()
        self._open[slot] = True
        self.frames_in[slot] = 0
        return slot

    def close(self, slot: int) -> None:
        import numpy as np
        if slot not in self._open:
            raise KeyError(f"slot {slot} is not open")
        del self._open[slot]
        self._buf[slot] = np.zeros(0, dtype=np.float32)
        self._free.append(slot)

    def push_pcm(self, slot: int, samples) -> None:
        import numpy as np
        if slot not in self._open:
            raise KeyError(f"slot {slot} is not open")
        samples = np.asarray(samples, dtype=np.float32).reshape(-1)
        if self._buf[slot].size + samples.size > self.max_samples:
            raise OverflowError(f"slot {slot}: more than {self.max_samples} samples buffered")
        self._buf[slot] = np.concatenate((self._buf[slot], samples))

    def buffered_frames(self, slot: int) -> int:
        return self._buf[slot].size // self.frame_size

    def next_frame(self, batch_pcm, updates) -> list[int]:
        """Fills ``batch_pcm`` f32 [B * frame_size] and ``updates`` i32 [B] in place; returns the slots that contributed."""
        fs = self.frame_size
        assert batch_pcm.size == self.batch_size * fs and updates.size == self.batch_size
        pcm = batch_pcm.reshape(self.batch_size, fs)
        ready = []
        for slot in range(self.batch_size):
            if slot in self._open and self._buf[slot].size >= fs:
                pcm[slot] = self._buf[slot][:fs]
                self._buf[slot] = self._buf[slot][fs:]
                updates[slot] = RESET if self._open[slot] else ACTIVE
                self._open[slot] = False
                self.frames_in[slot] += 1
                ready.append(slot)
            else:
                pcm[slot] = 0.0
                updates[slot] = NODATA
        return ready
