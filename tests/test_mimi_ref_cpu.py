"""CPU: the fp64 Mimi reference (tests/util.py MimiRef64) and the acceptance rule of tests/test_gpu_zz_mimi_ref.py.

``MimiRef64`` restates one Mimi streaming frame in float64, teacher-forced stage by stage on the taps of the implementation
under test.  Here the fp32 CPU oracle (oracle/mimi.py) plays the implementation, and two things are shown:

* The rule accepts a correct fp32 Mimi: the oracle passes at every checkpoint of 4 sessions over 2 fresh frames and 3 frames
  across the wrap of the 250-slot rings (rings filled with random entries of the magnitude the stream had, offsets set to 246,
  249, 250 and 500, i.e. no wrap, the frame that wraps, and two wrapped rings).  The constants (tests/util.py MIMI_C) are about
  twice what the oracle needs; both are printed.  Offsets stay at 500 and below here: the oracle's vectorised fp32 exp is one
  ulp off on one RoPE frequency, which at position 45 000 turns that pair by 2e-4 rad, far above fp32 rounding.
* The rule rejects a Mimi with a subtle bug: each mutant below is applied to the reference, and the named checkpoint must
  reject it in every affected row (for "attends to the overwritten key", the two rows whose ring has wrapped), both under the
  oracle's constants MIMI_C and under the wider constants MIMI_C_TC that tests/test_gpu_zz_mimi_ref.py applies to the 3xTF32
  kernels.  The narrowest margin is the tanh-approximate GELU, about 9 times its tolerance under either.
"""
import pytest
import torch

from moshi_b200.config import MimiConfig
from moshi_b200.synth import synth_mimi_state_dict
from oracle import scenarios
from oracle.mimi import MimiOracle
from tests.util import (MIMI_C, MIMI_C_TC, MimiRef64, mimi_c_needed, mimi_checkpoints, mimi_kind, mimi_ratios, rvq_unexcused, RVQ_GAP_BOUND)

CFG = MimiConfig()
B = 4
FRESH, WRAPPED = 2, 3
WRAP_OFFSETS = torch.tensor([246, 249, 250, 500])
TRS = ("encoder_transformer", "decoder_transformer")


@pytest.fixture(scope="module")
def sd():
    return synth_mimi_state_dict(CFG, seed=scenarios.MIMI_SEED)


def _rings(st, which):
    return [(ls.k.clone(), ls.v.clone()) for ls in st.layers]


def _wrap(orc: MimiOracle, g: torch.Generator) -> dict:
    """Random rings of the stream's magnitude (per layer and k / v) and offsets WRAP_OFFSETS in both oracle transformers;
    returns the rings written, for the reference's replays."""
    new = {}
    for which, st in zip(TRS, (orc.enc_tr, orc.dec_tr)):
        st.offsets[:] = WRAP_OFFSETS
        for li, ls in enumerate(st.layers):
            ls.offset[:] = WRAP_OFFSETS
            ls.end_offset[:] = WRAP_OFFSETS
            ls.k = torch.randn(ls.k.shape, generator=g) * ls.k[:, :, :4].pow(2).mean().sqrt()
            ls.v = torch.randn(ls.v.shape, generator=g) * ls.v[:, :, :4].pow(2).mean().sqrt()
            new[(which, li)] = (ls.k.clone(), ls.v.clone())
    return new


@pytest.fixture(scope="module")
def stream(sd):
    """The oracle over FRESH + WRAPPED frames.  Per frame: the inputs the reference needs (pcm, encoder taps and rings before,
    codes and latent, decoder taps and rings before), the oracle's rings after, the offsets before."""
    orc = MimiOracle(sd, CFG)
    orc.streaming(B)
    pcm = scenarios.mimi_noise(B, FRESH + WRAPPED, seed=31)
    g = torch.Generator().manual_seed(3)
    frames = []
    for f in range(FRESH + WRAPPED):
        if f == FRESH:
            _wrap(orc, g)
        x = pcm[..., f * 1920:(f + 1) * 1920]
        off = {w: st.layers[0].offset.clone() for w, st in zip(TRS, (orc.enc_tr, orc.dec_tr))}
        enc_rings = _rings(orc.enc_tr, TRS[0])
        orc.trace = {}
        lat = orc.encode_to_latent(x)
        codes = orc.quantize(lat)[..., 0]
        enc_taps = dict(orc.trace)
        dec_rings = _rings(orc.dec_tr, TRS[1])
        orc.trace = {}
        orc.decode(codes[..., None])
        dec_taps = dict(orc.trace)
        after = {}
        for which, st in zip(TRS, (orc.enc_tr, orc.dec_tr)):
            for li, ls in enumerate(st.layers):
                after[f"{which}.{li}.k"], after[f"{which}.{li}.v"] = ls.k.clone(), ls.v.clone()
        frames.append(dict(pcm=x, enc_taps=enc_taps, enc_rings=enc_rings, codes=codes, latent=lat[..., 0], dec_taps=dec_taps,
                           dec_rings=dec_rings, after=after, off=off))
    return frames


LAST_DEC = "dec.14"


def _replay(sd, frames, mutant=None) -> list:
    """MimiRef64 over the oracle's frames: per frame (checkpoints, RVQ verdict)."""
    ref = MimiRef64(sd, CFG, B, mutant)
    out = []
    for f, fr in enumerate(frames):
        if f == FRESH:
            for w in TRS:
                ref.offset[w] = WRAP_OFFSETS.clone()
        want = ref.encode_frame(fr["pcm"], fr["enc_taps"], fr["enc_rings"])
        q = ref.quantize(fr["latent"], fr["codes"])
        want.update(ref.decode_frame(fr["codes"], fr["dec_taps"], fr["dec_rings"]))
        taps = {**fr["enc_taps"], **fr["dec_taps"]}
        out.append((mimi_checkpoints(want, taps, fr["after"], fr["off"], torch.ones(B, dtype=torch.bool), CFG.tr_context), q))
    return out


@pytest.fixture(scope="module")
def reference(sd, stream):
    return _replay(sd, stream)


def test_fp32_oracle_passes_every_checkpoint(stream, reference):
    need = {}
    for f, (cps, q) in enumerate(reference):
        for name, got, want, per_head in cps:
            kind = mimi_kind(name, LAST_DEC)
            need[kind] = max(need.get(kind, 0.0), mimi_c_needed(got, want, per_head))
            r = mimi_ratios(got, want, MIMI_C[kind], per_head)
            assert (r <= 1).all(), (f, name, r)
        assert not rvq_unexcused(stream[f]["codes"], q, RVQ_GAP_BOUND).any(), f
        assert torch.equal(q["codes"], stream[f]["codes"]), f          # no near tie in these frames: the codes agree exactly
    print("\nc the fp32 oracle needs / c used:")
    for kind in sorted(need):
        print(f"  {kind:12s} {need[kind]:.2e} / {MIMI_C[kind]:.2e}")
        assert need[kind] <= MIMI_C[kind]


def _kblock(key: str, kb: int = 1, tap: int | None = 0):
    """State-dict weight ``key`` with input channels kb*32 .. kb*32+31 zeroed (at one tap of a conv)."""
    def f(k, w):
        if k != key:
            return w
        w = w.clone()
        if tap is None:
            w[:, kb * 32:(kb + 1) * 32] = 0
        else:
            w[:, kb * 32:(kb + 1) * 32, tap] = 0
        return w
    return {"weight": f}


E0 = "encoder_transformer"
WRAP = FRESH                 # the first frame across the ring wrap
ALL = list(range(B))
MUTANTS = {
    # name: (mutant, (frame, checkpoint) that must reject it, rows affected)
    "attention drops the oldest in-context key": ({"attn": {"drop_oldest": True}}, (WRAP, f"{E0}.1.k"), ALL),
    "attention attends to the key this step overwrote": ({"attn": {"overwritten": True}}, (WRAP, f"{E0}.1.k"), [2, 3]),
    "query 0 sees query 1's key": ({"attn": {"q0_sees_q1": True}}, (WRAP, f"{E0}.1.k"), ALL),
    "RoPE position off by one": ({"rope_shift": 1}, (WRAP, f"{E0}.0.k"), ALL),
    "layer scales swapped": ({"swap_layer_scales": True}, (WRAP, f"{E0}.1.k"), ALL),
    "tanh-approximate GELU": ({"gelu_tanh": True}, (WRAP, f"{E0}.1.k"), ALL),
    "LayerNorm variance over C - 1": ({"ln_unbiased": True}, (WRAP, f"{E0}.0.k"), ALL),
    "k-block missing: SEANet conv": (_kblock("encoder.model.3.conv.conv.weight"), (0, "enc.3"), ALL),
    "k-block missing: transformer linear1": (_kblock(f"{E0}.transformer.layers.0.linear1.weight", 5, None), (WRAP, f"{E0}.1.k"), ALL),
    "conv carried context shifted by one row": ({"conv_shift": "encoder.model.3.conv.conv"}, (1, "enc.3"), ALL),
    "ELU not applied to the activated copy": ({"no_elu": "encoder.model.6.conv.conv"}, (0, "enc.6"), ALL),
    "transposed-conv carry dropped": ({"no_carry": "decoder.model.2.convtr.convtr"}, (1, "dec.2"), ALL),
    "upsample carry dropped": ({"no_carry": "upsample.convtr.convtr.convtr"}, (1, "dec.up"), ALL),
    "RVQ level searched with the next level's codebook": ({"rvq_codebook_shift": ("rvq_rest", 2)}, (0, "codes"), ALL),
    "RVQ residual not updated": ({"rvq_no_residual": True}, (0, "codes"), ALL),
    "semantic and acoustic projections swapped": ({"rvq_swap_proj": True}, (0, "codes"), ALL),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_rejected_at_its_checkpoint_in_every_row(sd, stream, name):
    mutant, (frame, cp), rows = MUTANTS[name]
    cps, q = _replay(sd, stream[:frame + 1], mutant)[frame]
    if cp == "codes":
        r = rvq_unexcused(stream[frame]["codes"], q, RVQ_GAP_BOUND).sum(dim=1).double()       # unexcused codes per row
        print(f"{name}: rejected at frame {frame} codes, unexcused codes per row {r.tolist()}")
        assert (r[rows] > 0).all(), (name, r)
        return
    got, want, per_head = next((g, w, ph) for n, g, w, ph in cps if n == cp)
    kind = mimi_kind(cp, LAST_DEC)
    r = mimi_ratios(got, want, MIMI_C[kind], per_head)
    r_tc = mimi_ratios(got, want, MIMI_C_TC[kind], per_head)
    print(f"{name}: rejected at frame {frame} {cp}, row ratios {[f'{float(x):.3g}' for x in r]} "
          f"(under the 3xTF32 constants {[f'{float(x):.3g}' for x in r_tc]})")
    assert (r[rows] > 1).all(), (name, r)
    assert (r_tc[rows] > 1).all(), (name, r_tc)
