"""Wire protocol of the dialogue servers in front of the batched frame service (SURVEY.md 8f items 1 and 4).

Message framing: ``rust/protocol.md`` (one byte message type + payload inside each websocket binary message, little endian);
per-connection behaviour: ``moshi/moshi/server.py:74-152`` (incoming ``\\x01`` + opus bytes -> PCM -> 1920-sample frames ->
``mimi.encode -> lm_gen.step -> mimi.decode`` -> outgoing ``\\x01`` + opus bytes and ``\\x02`` + the text piece unless the
text token is 0 or 3 (padding), ``\\u2581`` replaced by a space).

Everything here is host logic and transport-agnostic: ``FrontEnd`` owns a ``SessionPool`` + a frame service
(``DialogueService`` on the GPU; any object with the same ``step`` in the CPU tests), connections push the websocket's binary
messages in and drain their outbox; one ``FrontEnd.step()`` per 80 ms runs ONE batched frame for every slot that has a frame
buffered.  The opus codec is the caller's (``sphn.OpusStreamReader / OpusStreamWriter`` in the reference: ``append_bytes(bytes)
-> float32 PCM`` and ``append_pcm(PCM) -> bytes``); ``RawPcmCodec`` is the same interface over raw little-endian float32
samples for the tests and for clients that skip opus.  ``serve_aiohttp`` binds it to an aiohttp websocket route like
``server.py:154-190``.
"""
from __future__ import annotations

import json
import math
import struct
import typing as tp
from dataclasses import dataclass, field

import numpy as np

from .serving import SessionPool

# rust/protocol.md
MT_HANDSHAKE, MT_AUDIO, MT_TEXT, MT_CONTROL, MT_METADATA, MT_ERROR, MT_PING = range(7)
CONTROL_START, CONTROL_END_TURN, CONTROL_PAUSE, CONTROL_RESTART = range(4)
PROTOCOL_VERSION = 0


@dataclass
class Message:
    kind: int
    payload: tp.Any = None      # handshake: (protocol_version, model_version); audio: bytes; text / error: str;
                                # control: int; metadata: dict; ping: None


def encode_message(msg: Message) -> bytes:
    k = msg.kind
    if k == MT_HANDSHAKE:
        proto, model = msg.payload
        return bytes([k]) + struct.pack("<II", proto, model)
    if k == MT_AUDIO:
        return bytes([k]) + bytes(msg.payload)
    if k in (MT_TEXT, MT_ERROR):
        return bytes([k]) + str(msg.payload).encode("utf8")
    if k == MT_CONTROL:
        if msg.payload not in (CONTROL_START, CONTROL_END_TURN, CONTROL_PAUSE, CONTROL_RESTART):
            raise ValueError(f"unknown control {msg.payload}")
        return bytes([k, msg.payload])
    if k == MT_METADATA:
        return bytes([k]) + json.dumps(msg.payload).encode("utf8")
    if k == MT_PING:
        return bytes([k])
    raise ValueError(f"unknown message type {k}")


def decode_message(data: bytes) -> Message | None:
    """``None`` for an empty message or an unknown type ("messages with an unknown message type should be discarded")."""
    if not data:
        return None
    k, body = data[0], data[1:]
    if k == MT_HANDSHAKE:
        if len(body) != 8:
            raise ValueError("handshake payload must be two u32")
        return Message(k, struct.unpack("<II", body))
    if k == MT_AUDIO:
        return Message(k, bytes(body))
    if k in (MT_TEXT, MT_ERROR):
        return Message(k, body.decode("utf8"))
    if k == MT_CONTROL:
        if len(body) != 1 or body[0] > CONTROL_RESTART:
            raise ValueError("control payload must be one byte in 0..3")
        return Message(k, body[0])
    if k == MT_METADATA:
        return Message(k, json.loads(body.decode("utf8")))
    if k == MT_PING:
        return Message(k)
    return None


class RawPcmCodec:
    """The reader / writer interface of ``sphn.OpusStreamReader`` / ``OpusStreamWriter`` over raw float32 little-endian PCM."""

    def __init__(self, sample_rate: int = 24000):
        self.sample_rate = sample_rate
        self._tail = b""

    def append_bytes(self, data: bytes) -> np.ndarray:
        data = self._tail + bytes(data)
        n = len(data) // 4 * 4
        self._tail = data[n:]
        return np.frombuffer(data[:n], dtype="<f4").astype(np.float32)

    def append_pcm(self, pcm: np.ndarray) -> bytes:
        return np.asarray(pcm, dtype="<f4").tobytes()


def opus_codec(sample_rate: int = 24000):
    """(reader, writer) of the reference's opus streams when ``sphn`` is installed (server.py:165-166), else raw PCM."""
    try:
        import sphn  # type: ignore
        return sphn.OpusStreamReader(sample_rate), sphn.OpusStreamWriter(sample_rate)
    except ImportError:
        return RawPcmCodec(sample_rate), RawPcmCodec(sample_rate)


# SessionConfigReq (rust/moshi-backend/src/stream_both.rs) query parameters -> the service's per-session settings
SESSION_CONFIG_KEYS = {"text_temperature": ("temp_text", float), "text_topk": ("top_k_text", int), "audio_temperature": ("temp", float),
                       "audio_topk": ("top_k", int), "pad_mult": ("pad_mult", float),
                       "repetition_penalty_context": ("repetition_context", int), "repetition_penalty": ("repetition_penalty", float)}
# MetaData field of each setting (the JSON the Rust server sends after the handshake)
_METADATA_NAMES = {v[0]: k for k, v in SESSION_CONFIG_KEYS.items()}


class SessionConfigError(ValueError):
    """A malformed or out-of-range session setting in a connection's query."""


def session_settings(config: tp.Mapping[str, tp.Any], defaults: tp.Mapping[str, tp.Any], history: int) -> dict[str, tp.Any]:
    """Every setting of a session from its ``SessionConfigReq`` (query strings or numbers): a missing key takes the handle-wide
    value (``defaults``: temp_text, temp, top_k_text, top_k; pad_mult 0, repetition_context 0, repetition_penalty 1), top-k
    values are clamped to the handle's and the repetition context to ``history`` (the tokens each session's history holds),
    unknown keys are ignored (max_steps, the seeds, email, ...).  SessionConfigError for a malformed value, a negative
    temperature or top-k below 1, a repetition context outside [0, 1024] or a penalty outside (0, 1000]."""
    out = dict(temp_text=float(defaults["temp_text"]), temp=float(defaults["temp"]), top_k_text=int(defaults["top_k_text"]),
               top_k=int(defaults["top_k"]), pad_mult=0.0, repetition_context=0, repetition_penalty=1.0)
    for key, (name, kind) in SESSION_CONFIG_KEYS.items():
        if key not in config or config[key] is None:
            continue
        raw = config[key]
        try:
            if isinstance(raw, bool) or (kind is int and isinstance(raw, float) and not raw.is_integer()):
                raise ValueError
            v = kind(raw.strip() if isinstance(raw, str) else raw)
        except (TypeError, ValueError):
            raise SessionConfigError(f"{key}: malformed value {raw!r}") from None
        if kind is float and not math.isfinite(v):
            raise SessionConfigError(f"{key}: {raw!r} is not finite")
        out[name] = v
    if out["temp_text"] < 0 or out["temp"] < 0:
        raise SessionConfigError("temperatures must be >= 0")
    if out["top_k_text"] < 1 or out["top_k"] < 1:
        raise SessionConfigError("top-k values must be >= 1")
    if not 0 <= out["repetition_context"] <= 1024:
        raise SessionConfigError(f"repetition_penalty_context {out['repetition_context']} outside [0, 1024]")
    if not 0 < out["repetition_penalty"] <= 1000:
        raise SessionConfigError(f"repetition_penalty {out['repetition_penalty']} outside (0, 1000]")
    out["top_k_text"] = min(out["top_k_text"], int(defaults["top_k_text"]))
    out["top_k"] = min(out["top_k"], int(defaults["top_k"]))
    out["repetition_context"] = min(out["repetition_context"], int(history))
    return out


def session_metadata(settings: tp.Mapping[str, tp.Any]) -> dict[str, tp.Any]:
    """The effective settings under the Rust server's ``MetaData`` field names."""
    return {_METADATA_NAMES[k]: v for k, v in settings.items()}


@dataclass
class Connection:
    slot: int
    reader: tp.Any
    writer: tp.Any
    outbox: list[bytes] = field(default_factory=list)
    frames_out: int = 0
    settings: dict | None = None       # the session's own sampling settings (connect(config)), None = the service-wide values


class FrontEnd:
    """Connections <-> session slots <-> one batched frame step (the in-process session manager of SURVEY.md 8f item 4)."""

    def __init__(self, service, batch_size: int, frame_size: int = 1920, tokens_per_slot: int = 9,
                 text_tokenizer=None, model_version: int = 0, codec_factory: tp.Callable[[], tuple] | None = None):
        self.service = service
        self.pool = SessionPool(batch_size, frame_size)
        self.frame_size, self.tokens_per_slot = frame_size, tokens_per_slot
        self.text_tokenizer = text_tokenizer
        self.model_version = model_version
        self.codec_factory = codec_factory or opus_codec
        self.connections: dict[int, Connection] = {}
        self._own_settings: set[int] = set()     # slots the service samples with a connection's own settings
        B = batch_size
        self._pcm_in = np.zeros(B * frame_size, dtype=np.float32)
        self._updates = np.zeros(B, dtype=np.int32)
        self._pcm_out = np.zeros((B, frame_size), dtype=np.float32)
        self._tok_out = np.zeros((B, tokens_per_slot), dtype=np.int64)
        self._flags = np.zeros(B, dtype=np.uint8)

    # ---- connection lifecycle (server.py:154-190: handshake first, then the receive loop) --------------------------------------
    def connect(self, config: tp.Mapping[str, tp.Any] | None = None) -> Connection:
        """A new connection on a free slot.  ``config``: the connection's ``SessionConfigReq`` (e.g. the websocket URL's query):
        on a service with per-session sampling (``DialogueService(session_sampling=N)``) the slot samples with those settings
        (``session_settings``) and the outbox gets an ``MT_METADATA`` message with the effective values after the handshake;
        SessionConfigError for a bad value, with no slot taken.  A service without it ignores the config, as it always did.
        Without a config a slot that a previous connection gave settings returns to the service-wide values."""
        history = int(getattr(self.service, "session_sampling", None) or 0)
        settings = None
        if config is not None and history > 0:
            settings = session_settings(config, self.service.sampling_defaults, history)
        slot = self.pool.open()            # raises RuntimeError when every slot is taken
        reader, writer = self.codec_factory()
        conn = Connection(slot, reader, writer, settings=settings)
        try:
            self._apply_settings(conn)
        except BaseException:
            self.pool.close(slot)          # a refused connection gives its slot back
            raise
        conn.outbox.append(encode_message(Message(MT_HANDSHAKE, (PROTOCOL_VERSION, self.model_version))))   # server.py:167
        if settings is not None:
            conn.outbox.append(encode_message(Message(MT_METADATA, session_metadata(settings))))
        self.connections[slot] = conn
        return conn

    def _apply_settings(self, conn: Connection) -> None:
        """The connection's settings onto its slot, every field of them, so that a slot never keeps a previous session's."""
        if conn.settings is not None:
            self.service.set_session_sampling(conn.slot, **conn.settings)
            self._own_settings.add(conn.slot)
        elif conn.slot in self._own_settings:
            self.service.set_session_sampling(conn.slot)
            self._own_settings.discard(conn.slot)

    def disconnect(self, conn: Connection) -> None:
        if conn.slot in self.connections:
            del self.connections[conn.slot]
            self.pool.close(conn.slot)

    def receive(self, conn: Connection, data: bytes) -> None:
        """One websocket binary message (server.py:109-148)."""
        msg = decode_message(data)
        if msg is None:
            return                          # empty or unknown kind: discarded (server.py:115-117, 149-150)
        if msg.kind == MT_AUDIO:
            pcm = conn.reader.append_bytes(msg.payload)
            if pcm.shape[-1]:
                self.pool.push_pcm(conn.slot, pcm)
        elif msg.kind == MT_CONTROL and msg.payload == CONTROL_RESTART:
            # a restarted turn is a recycled slot: its next frame carries RESET (batched_asr.py:154-158)
            self.pool.close(conn.slot)
            slot = self.pool.open()
            if slot != conn.slot:
                self.connections[slot] = self.connections.pop(conn.slot)
                conn.slot = slot
                self._apply_settings(conn)          # the connection keeps its settings on its new slot
        # handshake / text / metadata / ping from the client carry nothing the model consumes

    # ---- one 80 ms tick --------------------------------------------------------------------------------------------------------
    def step(self) -> int:
        """Runs one batched frame if any slot has one buffered; returns the number of slots that produced output."""
        ready = self.pool.next_frame(self._pcm_in, self._updates)
        if not ready:
            return 0
        self.service.step(self._pcm_in, self._pcm_out, self._tok_out, updates=self._updates, flags_out=self._flags)
        produced = 0
        for slot in ready:
            conn = self.connections.get(slot)
            if conn is None or not self._flags[slot]:
                continue                    # still inside the delay warm-up: step() "returned None" for this slot (server.py:141-143)
            opus_bytes = conn.writer.append_pcm(self._pcm_out[slot])
            if len(opus_bytes) > 0:
                conn.outbox.append(encode_message(Message(MT_AUDIO, opus_bytes)))          # server.py:85-87
            text_token = int(self._tok_out[slot, 0])
            if text_token not in (0, 3) and self.text_tokenizer is not None:               # server.py:88-93
                piece = self.text_tokenizer.id_to_piece(text_token).replace("▁", " ")
                conn.outbox.append(encode_message(Message(MT_TEXT, piece)))
            conn.frames_out += 1
            produced += 1
        return produced


async def serve_aiohttp(front: FrontEnd, host: str = "localhost", port: int = 8998, path: str = "/api/chat", tick_s: float = 0.08):
    """Binds ``FrontEnd`` to an aiohttp websocket route (the transport of ``server.py:154-190, 260-284``): one task per
    connection feeds ``receive`` and drains the outbox, one ticker task calls ``step`` every 80 ms."""
    import asyncio

    import aiohttp
    from aiohttp import web

    async def handle(request):
        ws = web.WebSocketResponse()
        await ws.prepare(request)
        try:
            # SessionConfigReq in the query string (the web client's sliders): no setting key, no per-session settings
            config = {k: v for k, v in request.query.items() if k in SESSION_CONFIG_KEYS}
            conn = front.connect(config or None)
        except (RuntimeError, SessionConfigError) as e:
            await ws.send_bytes(encode_message(Message(MT_ERROR, str(e))))
            await ws.close()
            return ws

        async def drain():
            while not ws.closed:
                while conn.outbox:
                    await ws.send_bytes(conn.outbox.pop(0))
                await asyncio.sleep(tick_s / 4)
        task = asyncio.create_task(drain())
        try:
            async for message in ws:
                if message.type == aiohttp.WSMsgType.BINARY:
                    front.receive(conn, message.data)
                elif message.type in (aiohttp.WSMsgType.ERROR, aiohttp.WSMsgType.CLOSED):
                    break
        finally:
            task.cancel()
            front.disconnect(conn)
        return ws

    async def ticker():
        while True:
            front.step()
            await asyncio.sleep(tick_s)

    app = web.Application()
    app.router.add_get(path, handle)
    runner = web.AppRunner(app)
    await runner.setup()
    await web.TCPSite(runner, host, port).start()
    await ticker()
