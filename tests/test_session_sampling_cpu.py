"""CPU: per-session sampling settings.  A numpy restatement of the text sampler of a session-sampling LM step (the Rust server's
behaviour, lm_generate_multistream.rs:142-175 and 247-255, as DESIGN.md states it), with known answers; the connection
front-end's query parsing, clamping, metadata, RESTART and slot recycling over a fake service; the Python-side checks."""
import numpy as np
import pytest

from moshi_b200 import protocol as P
from moshi_b200.serving import NODATA

PAD, SPECIAL_LOW = 3, 0
DEFAULT = None           # a row that follows the handle-wide values


def _special(t: int, card: int) -> bool:
    return t in (SPECIAL_LOW, PAD, card)


def penalty_window(ring: np.ndarray, count: int, context: int, card: int) -> list[int]:
    """The newest `context` non-special tokens of a history ring (slot count % N is the next), repeats included."""
    N = ring.shape[0]
    out = []
    for j in range(min(count, N)):
        if len(out) >= context:
            break
        t = int(ring[(count - 1 - j) % N])
        if 0 <= t < card and not _special(t, card):
            out.append(t)
    return out


def text_scores_ref(logits: np.ndarray, ring: np.ndarray, count: int, card: int, use_sampling: bool, temp: float,
                    st: dict | None) -> tuple[np.ndarray, bool]:
    """Steps 1-3 for one row: fp32 scores (penalised logits / temp + pad bias on sampling rows, penalised logits on greedy ones)
    and whether the row samples."""
    pen, ctx, pad = 1.0, 0, 0.0
    if st is not None:
        temp, pen, ctx, pad = st["temp_text"], st["repetition_penalty"], st["repetition_context"], st["pad_mult"]
    l = logits.astype(np.float32).copy()
    if pen != 1.0 and ctx > 0:
        p = np.float32(pen)
        for i in set(penalty_window(ring, count, ctx, card)):
            l[i] = l[i] / p if l[i] >= 0 else l[i] * p
    sampling = bool(use_sampling) and temp > 0
    if sampling:
        l = l / np.float32(temp)
        if pad != 0.0:
            l[PAD] = l[PAD] + np.float32(pad)
    return l, sampling


def text_sample_ref(logits: np.ndarray, noise: np.ndarray, ring: np.ndarray, count: np.ndarray, use_sampling: bool, temp: float,
                    top_k: int, settings: list, executed: np.ndarray | None = None, tie: float = 1e-5):
    """Steps 1-5 for B rows.  logits fp32 [B, card] (the bf16 values), noise [B, >= k], ring int32 [B, N], count [B]; settings[b]
    a dict of the seven settings or None.  Returns (tokens [B], stable [B], ring, count): `stable` is False where the two best
    ranks' p / noise lie within `tie` of each other (the device's fp32 softmax sum may order them either way)."""
    B, card = logits.shape
    ring, count = ring.copy(), count.copy()
    toks, stable = np.zeros(B, np.int64), np.ones(B, bool)
    for b in range(B):
        st = settings[b]
        s, sampling = text_scores_ref(logits[b], ring[b], int(count[b]), card, use_sampling, temp, st)
        order = np.lexsort((np.arange(card), -s.astype(np.float64)))          # (score desc, id asc)
        if not sampling:
            toks[b] = order[0]
        else:
            k = min(st["top_k_text"] if st is not None else top_k, card)
            top = order[:k]
            d = (s[top] - s.max()).astype(np.float64)
            r = np.exp(d) / noise[b, :k].astype(np.float64)
            j = int(np.argmax(r))
            toks[b] = top[j]
            if k > 1:
                two = np.sort(r)[-2:]
                stable[b] = two[1] > two[0] * (1 + tie)
        if (executed is None or executed[b]) and not _special(int(toks[b]), card):
            ring[b, count[b] % ring.shape[1]] = toks[b]
            count[b] += 1
    return toks, stable, ring, count


def settings(temp_text=0.7, temp=0.8, top_k_text=25, top_k=250, pad_mult=0.0, repetition_context=0, repetition_penalty=1.0):
    return dict(temp_text=temp_text, temp=temp, top_k_text=top_k_text, top_k=top_k, pad_mult=pad_mult,
                repetition_context=repetition_context, repetition_penalty=repetition_penalty)


# ---------------------------------------------------------------------------------------------------------------------------
# the restatement, known answers
# ---------------------------------------------------------------------------------------------------------------------------
def _ring(tokens: list[int], N: int = 8) -> tuple[np.ndarray, int]:
    r = np.full(N, -7, np.int32)
    for i, t in enumerate(tokens):
        r[i % N] = t
    return r, len(tokens)


def test_window_skips_special_ids_and_counts_repeats():
    card = 20
    ring, c = _ring([5, 6, 0, 7, 3, 7, 20, 9])                  # newest last: 9, (20), 7, (3), 7, (0), 6, 5
    assert penalty_window(ring, c, 3, card) == [9, 7, 7]       # repeats count, special ids neither count nor appear
    assert penalty_window(ring, c, 100, card) == [9, 7, 7, 6, 5]    # a window longer than the history takes all of it
    assert penalty_window(ring, c, 0, card) == []
    ring, c = _ring(list(range(4, 16)), N=8)                   # wrapped: only the newest 8 are kept
    assert penalty_window(ring, c, 100, card) == list(range(15, 7, -1))


def test_penalty_divides_positive_and_multiplies_negative_logits_once_per_id():
    card = 12
    l = np.array([0.5, 1, 2, 3, -1.5, 4, -2, 0, 1, 1, 1, 1], np.float32)
    ring, c = _ring([2, 4, 2, 4, 6, 7])
    s, sampling = text_scores_ref(l, ring, c, card, False, 0.7, settings(repetition_context=6, repetition_penalty=2.0))
    assert not sampling
    want = l.copy()
    want[2], want[4], want[6], want[7] = 1.0, -3.0, -4.0, 0.0          # 2 and 4 penalised once although repeated
    assert np.array_equal(s, want)
    # penalty 1 or context 0 changes nothing
    for st in (settings(repetition_context=6, repetition_penalty=1.0), settings(repetition_context=0, repetition_penalty=3.0)):
        assert np.array_equal(text_scores_ref(l, ring, c, card, False, 0.7, st)[0], l)


def test_greedy_row_with_penalty_ignores_pad_bias():
    card = 10
    l = np.zeros(card, np.float32)
    l[5], l[6], l[PAD] = 3.0, 2.0, 2.5
    ring, c = _ring([5])
    st = settings(temp_text=0.0, repetition_context=1, repetition_penalty=2.0, pad_mult=100.0)
    toks, _, ring2, c2 = text_sample_ref(l[None], np.ones((1, 25), np.float32), ring[None], np.array([c]), True, 0.7, 25, [st])
    assert toks[0] == PAD                    # 5 -> 1.5 after the penalty; pad at 2.5 wins, its bias ignored on a greedy row
    assert c2[0] == c                        # the padding token is not appended
    l[PAD] = 0.0
    toks, _, ring2, c2 = text_sample_ref(l[None], np.ones((1, 25), np.float32), ring[None], np.array([c]), True, 0.7, 25, [st])
    assert toks[0] == 6 and c2[0] == c + 1 and ring2[0, c % 8] == 6


def test_pad_bias_is_added_to_the_tempered_score():
    card = 10
    l = np.zeros(card, np.float32)
    l[4] = 1.4
    st = settings(temp_text=0.7, pad_mult=0.0)
    s, sampling = text_scores_ref(l, np.zeros(4, np.int32), 0, card, True, 0.7, st)
    assert sampling and s[4] == np.float32(1.4) / np.float32(0.7) and s[PAD] == 0
    st["pad_mult"] = 5.0
    s, _ = text_scores_ref(l, np.zeros(4, np.int32), 0, card, True, 0.7, st)
    assert s[PAD] == np.float32(5.0)
    noise = np.ones((1, 25), np.float32)
    toks, *_ = text_sample_ref(l[None], noise, np.zeros((1, 4), np.int32), np.zeros(1, np.int64), True, 0.7, 25, [st])
    assert toks[0] == PAD                    # exp(5) against exp(2): the biased pad is the most likely and noise is flat


def test_top_k_ranks_by_score_then_id_and_paused_rows_do_not_append():
    card = 8
    l = np.array([0, 0, 1, 1, 1, 0, 0, 0], np.float32)
    noise = np.array([[1.0, 0.5, 9.0]], np.float32)           # rank 1 (id 3) has the best p / noise among the top 2
    toks, *_ = text_sample_ref(l[None], noise, np.zeros((1, 4), np.int32), np.zeros(1, np.int64), True, 1.0, 2, [DEFAULT])
    assert toks[0] == 3
    toks, _, ring, cnt = text_sample_ref(l[None], noise, np.zeros((1, 4), np.int32), np.zeros(1, np.int64), True, 1.0, 2, [DEFAULT],
                                         executed=np.array([False]))
    assert toks[0] == 3 and cnt[0] == 0


# ---------------------------------------------------------------------------------------------------------------------------
# the front-end over a fake service
# ---------------------------------------------------------------------------------------------------------------------------
class SamplingService:
    """Records the settings given to each slot; one frame = PCM echoed, text token 5."""
    sampling_defaults = dict(temp_text=0.7, temp=0.8, top_k_text=25, top_k=250)
    session_sampling = 64                # tokens of text history per session

    def __init__(self, B):
        self.slot_settings = {b: None for b in range(B)}
        self.calls = []

    def set_session_sampling(self, slot, **settings):
        self.calls.append((slot, dict(settings)))
        self.slot_settings[slot] = dict(settings) if settings else None

    def step(self, batch_pcm, pcm_out, tokens_out, updates=None, flags_out=None, noise=None):
        for b in range(pcm_out.shape[0]):
            flags_out[b] = updates[b] != NODATA
            tokens_out[b] = 5


def _front(B=2):
    svc = SamplingService(B)
    return svc, P.FrontEnd(svc, B, 4, tokens_per_slot=2, codec_factory=lambda: (P.RawPcmCodec(), P.RawPcmCodec()))


def test_query_settings_clamped_and_metadata_sent():
    svc, front = _front()
    conn = front.connect({"text_temperature": "0.5", "text_topk": "400", "audio_topk": "100", "repetition_penalty": "1.5",
                          "repetition_penalty_context": "32", "max_steps": "9", "text_seed": "3", "email": "x", "zoom": "2"})
    want = dict(temp_text=0.5, temp=0.8, top_k_text=25, top_k=100, pad_mult=0.0, repetition_context=32, repetition_penalty=1.5)
    assert svc.slot_settings[conn.slot] == want
    assert P.decode_message(conn.outbox[0]).kind == P.MT_HANDSHAKE
    meta = P.decode_message(conn.outbox[1])
    assert meta.kind == P.MT_METADATA
    assert meta.payload == {"text_temperature": 0.5, "audio_temperature": 0.8, "text_topk": 25, "audio_topk": 100, "pad_mult": 0.0,
                            "repetition_penalty_context": 32, "repetition_penalty": 1.5}


@pytest.mark.parametrize("bad", [{"text_temperature": "hot"}, {"text_topk": "2.5"}, {"audio_topk": "0"}, {"text_temperature": "-1"},
                                 {"repetition_penalty": "0"}, {"repetition_penalty_context": "5000"}, {"pad_mult": "nan"},
                                 {"audio_temperature": "inf"}])
def test_malformed_or_out_of_range_values_are_refused_without_a_slot(bad):
    svc, front = _front()
    with pytest.raises(P.SessionConfigError):
        front.connect(bad)
    assert front.pool.free_slots == 2 and not svc.calls


def test_restart_keeps_settings_and_recycled_slots_get_full_settings():
    svc, front = _front(B=2)
    a = front.connect({"pad_mult": "2"})
    b = front.connect()                                        # no config: nothing set
    assert (a.slot, b.slot) == (0, 1)
    assert svc.calls == [(0, svc.slot_settings[0])] and svc.slot_settings[0]["pad_mult"] == 2.0
    front.disconnect(b)
    front.receive(a, P.encode_message(P.Message(P.MT_CONTROL, P.CONTROL_RESTART)))
    assert a.slot == 0 and svc.slot_settings[0]["pad_mult"] == 2.0       # the same slot back, its settings kept

    # a pool that hands a restarted connection another slot: the settings follow the connection there
    close = front.pool.close

    def close_to_bottom(slot):
        close(slot)
        front.pool._free.insert(0, front.pool._free.pop())
    front.pool.close = close_to_bottom
    front.receive(a, P.encode_message(P.Message(P.MT_CONTROL, P.CONTROL_RESTART)))
    assert a.slot == 1 and front.connections[1] is a
    assert svc.slot_settings[1] == svc.slot_settings[0] and svc.slot_settings[1]["pad_mult"] == 2.0
    front.pool.close = close

    c = front.connect({"text_temperature": "0.1"})             # slot 0, configured by a's first session: a full new setting
    assert c.slot == 0
    assert svc.slot_settings[0] == dict(temp_text=0.1, temp=0.8, top_k_text=25, top_k=250, pad_mult=0.0, repetition_context=0,
                                        repetition_penalty=1.0)
    front.disconnect(a)
    d = front.connect()                                        # slot 1, configured by a: back to the service-wide values
    assert d.slot == 1 and svc.slot_settings[1] is None and svc.calls[-1] == (1, {})


# the query the reference web client appends to every /api/chat connection (Conversation.tsx)
WEB_CLIENT_QUERY = {"text_temperature": "0.7", "text_topk": "25", "audio_temperature": "0.8", "audio_topk": "250", "pad_mult": "0",
                    "repetition_penalty_context": "64", "repetition_penalty": "1.0"}


class PlainService(SamplingService):
    """A service without per-session sampling, whose set_session_sampling refuses like LMGen's does."""
    session_sampling = None

    def set_session_sampling(self, slot, **settings):
        raise RuntimeError("per-session sampling is off")


def test_service_without_the_feature_ignores_the_web_client_query():
    svc = PlainService(2)
    front = P.FrontEnd(svc, 2, 4, tokens_per_slot=2, codec_factory=lambda: (P.RawPcmCodec(), P.RawPcmCodec()))
    for _ in range(5):                                         # as before: connected, settings dropped, no metadata, no leak
        conn = front.connect(dict(WEB_CLIENT_QUERY))
        assert [P.decode_message(m).kind for m in conn.outbox] == [P.MT_HANDSHAKE]
        front.disconnect(conn)
    assert front.pool.free_slots == 2


def test_a_refused_setting_gives_the_slot_back():
    svc = PlainService(2)
    svc.session_sampling = 32                                  # claims the feature, then refuses
    front = P.FrontEnd(svc, 2, 4, tokens_per_slot=2, codec_factory=lambda: (P.RawPcmCodec(), P.RawPcmCodec()))
    for _ in range(3):
        with pytest.raises(RuntimeError):
            front.connect(dict(WEB_CLIENT_QUERY))
    assert front.pool.free_slots == 2 and not front.connections


def test_repetition_context_is_clamped_to_the_history():
    svc, front = _front()
    conn = front.connect({"repetition_penalty_context": "200", "repetition_penalty": "1.3"})
    assert svc.slot_settings[conn.slot]["repetition_context"] == 64
    assert P.decode_message(conn.outbox[1]).payload["repetition_penalty_context"] == 64


def test_front_end_without_config_never_touches_settings():
    svc, front = _front()
    a = front.connect()
    assert len(a.outbox) == 1 and not svc.calls
    front.receive(a, P.encode_message(P.Message(P.MT_AUDIO, np.zeros(4, "<f4").tobytes())))
    assert front.step() == 1 and not svc.calls


# ---------------------------------------------------------------------------------------------------------------------------
# Python-side checks
# ---------------------------------------------------------------------------------------------------------------------------
def test_session_settings_defaults_and_types():
    d = SamplingService.sampling_defaults
    assert P.session_settings({}, d, 64) == dict(temp_text=0.7, temp=0.8, top_k_text=25, top_k=250, pad_mult=0.0, repetition_context=0,
                                              repetition_penalty=1.0)
    assert P.session_settings({"text_topk": 7, "audio_temperature": 0}, d, 64)["top_k_text"] == 7
    for bad in ({"text_topk": True}, {"text_topk": 2.5}, {"pad_mult": "x"}):
        with pytest.raises(P.SessionConfigError):
            P.session_settings(bad, d, 64)


def test_lmgen_set_session_sampling_checks_before_the_library():
    from moshi_b200.models.lm import LMGen
    g = LMGen.__new__(LMGen)
    g._batch, g.session_sampling = None, 8
    with pytest.raises(AssertionError):
        g.set_session_sampling([0], temp=0.5)
    g._batch, g.session_sampling = 2, None
    with pytest.raises(RuntimeError):
        g.set_session_sampling([0], temp=0.5)
    g.session_sampling = 8
    with pytest.raises(ValueError):
        g.set_session_sampling([2], temp=0.5)
    with pytest.raises(ValueError):
        g.set_session_sampling([0], top_k=2.5)
