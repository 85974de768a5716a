"""``MimiModel`` with the reference's public surface, backed by the sm_90a library.

Mirrors ``moshi/moshi/models/compression.py:97-433`` (properties, ``encode`` / ``decode`` /
``encode_to_latent`` / ``decode_latent``) and the ``StreamingModule`` protocol of
``moshi/moshi/modules/streaming.py:54-211`` (``streaming`` / ``streaming_forever`` /
``reset_streaming`` / ``set_exec_mask``).  torch tensors are only owners of device memory here; all
arithmetic happens in ``libmoshi_b200.so``.
"""
from __future__ import annotations

import ctypes as C
import typing as tp
from contextlib import ExitStack
from types import SimpleNamespace

import torch

from .. import _lib
from ..config import MimiConfig
from .state_dict import normalize_mimi_state_dict


def _config_struct(cfg: MimiConfig) -> _lib.MimiConfigC:
    c = _lib.MimiConfigC()
    c.sample_rate, c.frame_rate, c.channels = cfg.sample_rate, cfg.frame_rate, cfg.channels
    c.dimension, c.n_filters, c.n_residual_layers = cfg.dimension, cfg.n_filters, cfg.n_residual_layers
    c.n_ratios = len(cfg.ratios)
    for i, r in enumerate(cfg.ratios):
        c.ratios[i] = r
    c.kernel_size, c.residual_kernel_size = cfg.kernel_size, cfg.residual_kernel_size
    c.last_kernel_size, c.dilation_base, c.compress = cfg.last_kernel_size, cfg.dilation_base, cfg.compress
    c.tr_d_model, c.tr_num_heads, c.tr_num_layers = cfg.tr_d_model, cfg.tr_num_heads, cfg.tr_num_layers
    c.tr_dim_feedforward, c.tr_context, c.tr_max_period = cfg.tr_dim_feedforward, cfg.tr_context, cfg.tr_max_period
    c.q_dimension, c.q_bins, c.q_n_q, c.q_n_semantic = cfg.q_dimension, cfg.q_bins, cfg.q_n_q, cfg.q_n_semantic
    c.num_codebooks = cfg.num_codebooks
    return c


class MimiModel:
    """Mimi on one GPU.  Construct through ``loaders.get_mimi``."""

    def __init__(self, cfg: MimiConfig, state_dict: tp.Mapping[str, torch.Tensor],
                 device: torch.device | str = "cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("moshi_b200.MimiModel runs on a CUDA device only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.lib()
        self._h = C.c_void_p()
        self._batch: int | None = None
        self._num_codebooks = cfg.num_codebooks
        self.use_graph = True      # replay each one-frame encode / decode as a CUDA graph
        # carried input rows per SEANet layer (state-dict prefix of its nn.Conv1d / nn.ConvTranspose1d -> P): StreamingConv1d keeps
        # (k - 1) * dilation + 1 - stride samples (conv.py:233-243), a transposed conv its previous input step
        from ..synth import seanet_layout
        self._carried_rows: dict[str, int] = {}
        for side, layers in zip(("encoder", "decoder"), seanet_layout(cfg)):
            for kind, idx, cin, cout, k, stride, dil in layers:
                base = f"{side}.model.{idx}"
                if kind == "conv":
                    self._carried_rows[base + ".conv.conv"] = (k - 1) * dil + 1 - stride
                elif kind == "convtr":
                    self._carried_rows[base + ".convtr.convtr"] = 1
                else:
                    self._carried_rows[base + ".block.1.conv.conv"] = (k - 1) * dil
                    self._carried_rows[base + ".block.3.conv.conv"] = 0
        with torch.cuda.device(self.device):
            _lib.check(self._lib.b200_mimi_create(C.byref(_config_struct(cfg)), C.byref(self._h)))
            for name, t in normalize_mimi_state_dict(state_dict).items():
                if not t.dtype.is_floating_point:
                    continue
                t = t.detach().to(device=self.device, dtype=torch.float32).contiguous()
                shape = (C.c_int64 * t.dim())(*t.shape)
                _lib.check(self._lib.b200_mimi_load_tensor(self._h, name.encode(), _lib.ptr(t), _lib.B200_F32,
                                                           t.dim(), shape))
            _lib.check(self._lib.b200_mimi_finalize(self._h))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self._lib.b200_mimi_destroy(h)
            except Exception:
                pass
            self._h = C.c_void_p()

    # ---- properties (compression.py:240-275) ----------------------------------------------------
    @property
    def channels(self) -> int:
        return self.cfg.channels

    @property
    def frame_rate(self) -> float:
        return self.cfg.frame_rate

    @property
    def sample_rate(self) -> int:
        return self.cfg.sample_rate

    @property
    def frame_size(self) -> int:
        return self.cfg.frame_size

    @property
    def dimension(self) -> int:
        return self.cfg.dimension

    @property
    def total_codebooks(self) -> int:
        return self.cfg.q_n_q

    @property
    def num_codebooks(self) -> int:
        return self._num_codebooks

    @property
    def cardinality(self) -> int:
        return self.cfg.q_bins

    def set_num_codebooks(self, n: int) -> None:
        _lib.check(self._lib.b200_mimi_set_num_codebooks(self._h, int(n)))
        self._num_codebooks = int(n)

    def eval(self) -> "MimiModel":
        return self

    # ---- streaming protocol (streaming.py:131-211) ----------------------------------------------
    @property
    def is_streaming(self) -> bool:
        return self._batch is not None

    def _start(self, batch_size: int) -> None:
        assert self._batch is None, "mimi is already streaming!"          # streaming.py:112
        with torch.cuda.device(self.device):
            _lib.check(self._lib.b200_mimi_set_graph(self._h, int(self.use_graph)))
            _lib.check(self._lib.b200_mimi_streaming_begin(self._h, int(batch_size), _lib.current_stream(self.device)))
        self._batch = int(batch_size)

    def _stop(self) -> None:
        if self._batch is not None:
            self._lib.b200_mimi_streaming_end(self._h)
            self._batch = None

    def streaming(self, batch_size: int) -> ExitStack:
        stack = ExitStack()
        self._start(batch_size)
        stack.callback(self._stop)
        return stack

    def streaming_forever(self, batch_size: int) -> None:
        self._start(batch_size)

    def _mask(self, mask: torch.Tensor) -> torch.Tensor:
        assert self._batch is not None
        mask = mask.to(device=self.device, dtype=torch.bool).contiguous()
        assert mask.shape == (self._batch,), f"mask must have shape ({self._batch},)"
        return mask

    def reset_streaming(self, reset_mask: torch.Tensor | None = None) -> None:
        assert self._batch is not None, "Trying to reset streaming, but mimi wasn't streaming."
        m = None if reset_mask is None else self._mask(reset_mask)
        _lib.check(self._lib.b200_mimi_reset(self._h, _lib.ptr(m)))

    def set_exec_mask(self, exec_mask: torch.Tensor) -> None:
        assert self._batch is not None
        m = self._mask(exec_mask)
        _lib.check(self._lib.b200_mimi_set_exec_mask(self._h, _lib.ptr(m)))

    # ---- one session ----------------------------------------------------------------------------------
    def export_session(self, row: int) -> torch.Tensor:
        """Encoder and decoder state of session ``row`` as a uint8 record on the model's device (``b200_mimi_session_export``,
        fixed size per configuration).  The row is not changed."""
        assert self._batch is not None, "mimi is not streaming"
        n = C.c_int64()
        _lib.check(self._lib.b200_mimi_session_bytes(self._h, C.byref(n)))
        rec = torch.empty(n.value, dtype=torch.uint8, device=self.device)
        _lib.check(self._lib.b200_mimi_session_export(self._h, int(row), _lib.ptr(rec), n.value))
        return rec

    def import_session(self, row: int, record: torch.Tensor) -> None:
        """Replaces session ``row`` with a record of ``export_session`` from a handle of the same configuration, on any device.
        Nothing changes if it is refused (ValueError for an incompatible record or row)."""
        assert self._batch is not None, "mimi is not streaming"
        rec = record.to(self.device).contiguous()
        assert rec.dtype == torch.uint8 and rec.dim() == 1, "a session record is a 1-d uint8 tensor"
        _lib.check(self._lib.b200_mimi_session_import(self._h, int(row), _lib.ptr(rec), rec.numel()))

    # ---- streaming state ------------------------------------------------------------------------------
    def _state_entries(self) -> list[tuple[str, torch.dtype, tuple[int, ...], int]]:
        from .lm import _TORCH_DTYPES
        out = []
        for i in range(int(self._lib.b200_mimi_state_count(self._h))):
            name, dt, nd, nb = C.c_char_p(), C.c_int(), C.c_int(), C.c_int64()
            shape = (C.c_int64 * 8)()
            _lib.check(self._lib.b200_mimi_state_entry(self._h, i, C.byref(name), C.byref(dt), C.byref(nd), shape, C.byref(nb)))
            out.append((name.value.decode(), _TORCH_DTYPES[dt.value], tuple(shape[:nd.value]), nb.value))
        return out

    @staticmethod
    def _split_tf32(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """x = hi + lo with hi = tf32(x), lo = tf32(x - hi), round-to-nearest (ties away): what the kernels' epilogues write."""
        def rna(t):
            return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
        hi = rna(x.float())
        return hi, rna(x.float() - hi)

    def get_streaming_state(self) -> dict[str, tp.Any]:
        """``StreamingModule.get_streaming_state`` (streaming.py:158-166): module path -> state object with the reference's field
        names.  StreamingConv1d: ``previous [B, Cin, P]``, ``first`` (conv.py:161-169); StreamingConvTranspose1d: the library
        carries the previous INPUT step instead of the overlap-add ``partial`` (the same information before the last matrix
        product, conv.py:349-361), reported as ``previous_input [B, Cin, 1]``; ``_MHAState``: ``kv_cache.cache [2, B, H, 250, 64]``,
        ``kv_cache.end_offset``, ``offset`` (transformer.py:196-288, 321-334); the depth-wise up-sampling keeps ``partial``.
        Tensors are copies."""
        assert self._batch is not None, "mimi is not streaming"
        with torch.cuda.device(self.device):
            raw = {}
            for name, dt, shape, nb in self._state_entries():
                t = torch.empty(shape, dtype=dt, device=self.device)
                _lib.check(self._lib.b200_mimi_state_read(self._h, name.encode(), _lib.ptr(t), nb))
                raw[name] = t
        B = self._batch
        mask = raw["exec_mask"].bool()
        state: dict[str, tp.Any] = {"": SimpleNamespace(batch_size=B, device=self.device, exec_mask=mask)}
        for name in raw:
            if not name.endswith(".ext_hi"):
                continue
            base = name[:-len(".ext_hi")]                          # e.g. encoder.model.3.conv.conv
            lo = raw.get(base + ".ext_lo")
            full = raw[name] if lo is None else raw[name] + lo     # [B, P + T, Cin]
            is_tr = base.endswith(".convtr.convtr")
            module = base[:-len(".convtr.convtr")] if is_tr else base[:-len(".conv.conv")]
            P = self._carried_rows[base]
            prev = full[:, :P].transpose(1, 2).contiguous()        # [B, Cin, P]
            # _raw: the carried rows exactly as the kernels hold them (re-splitting hi + lo is not always bit-identical)
            rawp = (raw[name][:, :P].clone(), None if lo is None else lo[:, :P].clone())
            if is_tr:
                state[module] = SimpleNamespace(batch_size=B, exec_mask=mask, previous_input=prev, _raw=rawp)
            else:
                state[module] = SimpleNamespace(batch_size=B, exec_mask=mask, previous=prev, _raw=rawp,
                                                first=torch.zeros(B, dtype=torch.bool, device=self.device))
        state["downsample.conv"] = SimpleNamespace(batch_size=B, exec_mask=mask, previous=raw["downsample.previous"],
                                                   first=raw["downsample.first"].bool())
        state["upsample.convtr"] = SimpleNamespace(batch_size=B, exec_mask=mask, partial=raw["upsample.partial"])
        for tr in ("encoder_transformer", "decoder_transformer"):
            off = raw[tr + ".offset"]
            state[tr + ".transformer"] = SimpleNamespace(batch_size=B, exec_mask=mask, offsets=off.clone())
            for i in range(self.cfg.tr_num_layers):
                kv = SimpleNamespace(cache=torch.stack([raw[f"{tr}.layers.{i}.k"], raw[f"{tr}.layers.{i}.v"]]), end_offset=off.clone())
                state[f"{tr}.transformer.layers.{i}.self_attn"] = SimpleNamespace(batch_size=B, exec_mask=mask, kv_cache=kv,
                                                                                 offset=off.clone())
        return state

    def set_streaming_state(self, state: dict[str, tp.Any]) -> None:
        """``set_streaming_state`` (streaming.py:168-181): every module state must be present and nothing else."""
        assert self._batch is not None, "mimi is not streaming"
        state = dict(state)
        entries = {name: (dt, shape, nb) for name, dt, shape, nb in self._state_entries()}

        def take(name):
            if name not in state:
                raise RuntimeError(f"Expected to find a streaming state for {name}.")
            return state.pop(name)

        def write(name, t):
            dt, shape, nb = entries[name]
            t = t.to(device=self.device, dtype=dt).contiguous()
            assert tuple(t.shape) == shape, (name, tuple(t.shape), shape)
            _lib.check(self._lib.b200_mimi_state_write(self._h, name.encode(), _lib.ptr(t), nb))

        with torch.cuda.device(self.device):
            root = take("")
            assert root.batch_size == self._batch, "snapshot was taken with another batch size"
            write("exec_mask", root.exec_mask.to(torch.uint8))
            for name, (dt, shape, nb) in entries.items():
                if not name.endswith(".ext_hi"):
                    continue
                base = name[:-len(".ext_hi")]
                is_tr = base.endswith(".convtr.convtr")
                st = take(base[:-len(".convtr.convtr")] if is_tr else base[:-len(".conv.conv")])
                prev = (st.previous_input if is_tr else st.previous).to(self.device).float().transpose(1, 2)   # [B, P, Cin]
                P = self._carried_rows[base]
                cur = torch.empty(shape, dtype=dt, device=self.device)
                _lib.check(self._lib.b200_mimi_state_read(self._h, name.encode(), _lib.ptr(cur), nb))
                rawp = getattr(st, "_raw", None)
                if rawp is not None and torch.equal((rawp[0] if rawp[1] is None else rawp[0] + rawp[1]), prev):
                    hi, lo = rawp                              # untouched snapshot: restore bit for bit
                elif base + ".ext_lo" in entries:
                    hi, lo = self._split_tf32(prev)
                else:
                    hi, lo = prev, None
                if base + ".ext_lo" in entries:
                    cur_lo = torch.empty(shape, dtype=dt, device=self.device)
                    _lib.check(self._lib.b200_mimi_state_read(self._h, (base + ".ext_lo").encode(), _lib.ptr(cur_lo), nb))
                    cur_lo[:, :P] = lo
                    write(base + ".ext_lo", cur_lo)
                cur[:, :P] = hi
                write(name, cur)
            st = take("downsample.conv")
            write("downsample.previous", st.previous)
            write("downsample.first", st.first.to(torch.uint8))
            write("upsample.partial", take("upsample.convtr").partial)
            for tr in ("encoder_transformer", "decoder_transformer"):
                write(tr + ".offset", take(tr + ".transformer").offsets.long())
                for i in range(self.cfg.tr_num_layers):
                    st = take(f"{tr}.transformer.layers.{i}.self_attn")
                    write(f"{tr}.layers.{i}.k", st.kv_cache.cache[0])
                    write(f"{tr}.layers.{i}.v", st.kv_cache.cache[1])
        if state:
            raise RuntimeError(f"Some states were not consumed: {list(state.keys())}")

    # ---- data path ------------------------------------------------------------------------------
    def _check_pcm(self, x: torch.Tensor) -> torch.Tensor:
        assert x.dim() == 3, f"expected audio of shape [B, C, T] but got {tuple(x.shape)}"
        assert x.shape[1] == self.channels
        return x.to(device=self.device, dtype=torch.float32).contiguous()

    def _with_session(self, batch: int):
        """Non-streaming calls run on a throw-away streaming session (fresh zero state), which is
        what the reference's ``state is None`` branch computes (conv.py:249-251, transformer.py:538-545)."""
        stack = ExitStack()
        if self._batch is None:
            stack.enter_context(self.streaming(batch))
        return stack

    def _encode_to_unquantized_latent(self, x: torch.Tensor) -> torch.Tensor:
        x = self._check_pcm(x)
        fs = self.frame_size
        if self._batch is None:
            extra = (-x.shape[-1]) % fs                                   # pad_for_conv1d, compression.py:358
            if extra:
                x = torch.nn.functional.pad(x, (0, extra))
        elif x.shape[-1] % fs != 0 or x.shape[-1] == 0:
            raise RuntimeError(
                f"Invalid input x of length {x.shape[-1]}. The length must be "
                f"a positive multiple of the frame size {fs}. "
                "You are responsible for buffering accordingly before feeding audio to Mimi.")
        n = x.shape[-1] // fs
        with self._with_session(x.shape[0]):
            assert x.shape[0] == self._batch, f"Got a batch size {x.shape[0]}, expected {self._batch}"
            out = torch.empty(x.shape[0], self.dimension, n, device=self.device, dtype=torch.float32)
            _lib.check(self._lib.b200_mimi_encode_to_latent(self._h, _lib.ptr(x), n, _lib.ptr(out)))
        return out

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        """f32 [B, 1, T] -> i64 [B, K, T / frame_size]  (compression.py:376-388)."""
        x = self._check_pcm(x)
        fs = self.frame_size
        if self._batch is None:
            extra = (-x.shape[-1]) % fs
            if extra:
                x = torch.nn.functional.pad(x, (0, extra))
        elif x.shape[-1] % fs != 0 or x.shape[-1] == 0:
            raise RuntimeError(
                f"Invalid input x of length {x.shape[-1]}. The length must be "
                f"a positive multiple of the frame size {fs}. "
                "You are responsible for buffering accordingly before feeding audio to Mimi.")
        n = x.shape[-1] // fs
        with self._with_session(x.shape[0]):
            assert x.shape[0] == self._batch, f"Got a batch size {x.shape[0]}, expected {self._batch}"
            codes = torch.empty(x.shape[0], self.num_codebooks, n, device=self.device, dtype=torch.int64)
            _lib.check(self._lib.b200_mimi_encode(self._h, _lib.ptr(x), n, _lib.ptr(codes)))
        return codes

    def encode_to_latent(self, x: torch.Tensor, quantize: bool = True) -> torch.Tensor:
        emb = self._encode_to_unquantized_latent(x)
        if not quantize:
            return emb
        with self._with_session(emb.shape[0]):
            codes = torch.empty(emb.shape[0], self.num_codebooks, emb.shape[-1], device=self.device, dtype=torch.int64)
            _lib.check(self._lib.b200_mimi_quantize(self._h, _lib.ptr(emb), emb.shape[-1], _lib.ptr(codes)))
        return self.decode_latent(codes)

    def _check_codes(self, codes: torch.Tensor) -> torch.Tensor:
        assert codes.dim() == 3, f"expected codes of shape [B, K, T] but got {tuple(codes.shape)}"
        assert not codes.dtype.is_floating_point, f"Codes should be integers, got {codes.dtype}"
        return codes.to(device=self.device, dtype=torch.int64).contiguous()

    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        """i64 [B, K, T] -> f32 [B, 1, T * frame_size]  (compression.py:406-429)."""
        codes = self._check_codes(codes)
        B, K, n = codes.shape
        with self._with_session(B):
            assert B == self._batch, f"Got a batch size {B}, expected {self._batch}"
            out = torch.empty(B, 1, n * self.frame_size, device=self.device, dtype=torch.float32)
            _lib.check(self._lib.b200_mimi_decode(self._h, _lib.ptr(codes), K, n, _lib.ptr(out)))
        return out

    def decode_latent(self, codes: torch.Tensor) -> torch.Tensor:
        codes = self._check_codes(codes)
        B, K, n = codes.shape
        with self._with_session(B):
            out = torch.empty(B, self.dimension, n, device=self.device, dtype=torch.float32)
            _lib.check(self._lib.b200_mimi_decode_latent(self._h, _lib.ptr(codes), K, n, _lib.ptr(out)))
        return out

    # ---- host-buffer entry points (bench.py e2e) --------------------------------------------------
    def encode_host(self, pcm_cpu: torch.Tensor, codes_cpu: torch.Tensor) -> None:
        n = pcm_cpu.shape[-1] // self.frame_size
        _lib.check(self._lib.b200_mimi_encode_host(self._h, _lib.ptr(pcm_cpu), n, _lib.ptr(codes_cpu)))

    def decode_host(self, codes_cpu: torch.Tensor, pcm_cpu: torch.Tensor) -> None:
        B, K, n = codes_cpu.shape
        _lib.check(self._lib.b200_mimi_decode_host(self._h, _lib.ptr(codes_cpu), K, n, _lib.ptr(pcm_cpu)))

    # ---- debugging / measurement -------------------------------------------------------------------
    def debug_buffer(self, name: str) -> torch.Tensor:
        """Copy of a named intermediate of the last encode/decode call (flat fp32)."""
        n = C.c_int64()
        _lib.check(self._lib.b200_mimi_read_buffer(self._h, name.encode(), None, 0, C.byref(n)))
        out = torch.empty(n.value, device=self.device, dtype=torch.float32)
        _lib.check(self._lib.b200_mimi_read_buffer(self._h, name.encode(), _lib.ptr(out), n.value, C.byref(n)))
        return out

    def algorithmic_bytes(self) -> int:
        return int(self._lib.b200_mimi_algorithmic_bytes(self._h))
