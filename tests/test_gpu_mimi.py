"""GPU: Mimi streaming encode / decode through the reference-shaped API against the CPU oracle and
the golden fixtures recorded from the unmodified reference."""
import pytest
import torch
from safetensors.torch import load_file

from moshi_b200.config import MimiConfig
from moshi_b200.synth import synth_mimi_state_dict
from oracle import scenarios
from oracle.mimi import MimiOracle
from tests.util import rvq_mismatches, stats

pytestmark = pytest.mark.gpu

LATENT_ATOL = 2e-4      # fp32 accumulation-order noise through ~40 layers; latent std ~0.8
PCM_ATOL = 5e-4         # north_star: PCM within a stated fp tolerance; PCM std ~1


@pytest.fixture(scope="module")
def sd():
    return synth_mimi_state_dict(MimiConfig(), seed=scenarios.MIMI_SEED)


@pytest.fixture(scope="module")
def gpu(sd):
    from moshi_b200.models import MimiModel
    return MimiModel(MimiConfig(), sd, device="cuda")


def _token_major(t: torch.Tensor) -> torch.Tensor:
    return t.transpose(1, 2).contiguous()


def test_properties_match_reference(gpu):
    assert (gpu.sample_rate, gpu.frame_rate, gpu.frame_size, gpu.channels) == (24000, 12.5, 1920, 1)
    assert (gpu.cardinality, gpu.num_codebooks, gpu.total_codebooks) == (2048, 8, 32)


@torch.no_grad()
def test_layer_by_layer_first_frames(gpu, sd):
    """Localises any divergence: every SEANet module output, both transformers, latent, PCM."""
    cfg = MimiConfig()
    orc = MimiOracle(sd, cfg)
    B = 2
    pcm = scenarios.mimi_noise(B, 3, seed=11)
    orc.streaming(B)
    report = []
    worst = 0.0
    with gpu.streaming(B):
        for f in range(3):
            x = pcm[..., f * 1920:(f + 1) * 1920]
            orc.trace = {}
            lat_o = orc.encode_to_latent(x)
            codes_o = orc.quantize(lat_o)
            pcm_o = orc.decode(codes_o)
            lat_g = gpu._encode_to_unquantized_latent(x.cuda())
            pcm_g = gpu.decode(codes_o.cuda())
            for name, want in orc.trace.items():
                if name in ("enc.14", "enc.tr", "dec.up", "dec.tr"):
                    want = _token_major(want)
                elif name in ("enc.latent", "dec.latent"):
                    want = want[..., 0]
                try:
                    got = gpu.debug_buffer(name).view(want.shape).cpu()
                except ValueError:
                    continue
                rel = (got - want).abs().max().item() / (want.abs().max().item() + 1e-30)
                worst = max(worst, rel)
                report.append(f"frame {f} {stats(name, got, want)}")
            report.append(f"frame {f} {stats('latent', lat_g, lat_o)}")
            report.append(f"frame {f} {stats('pcm', pcm_g, pcm_o)}")
            torch.testing.assert_close(lat_g.cpu(), lat_o, rtol=0, atol=LATENT_ATOL, msg="\n".join(report))
            torch.testing.assert_close(pcm_g.cpu(), pcm_o, rtol=0, atol=PCM_ATOL, msg="\n".join(report))
    print("\n".join(report))
    assert worst < 1e-3, "\n".join(report)


@torch.no_grad()
def test_rvq_kernel_is_exact_on_the_oracle_latent(gpu, sd):
    """Isolates the nearest-codebook search from encoder numerics (SURVEY.md 7 'minimum slice')."""
    orc = MimiOracle(sd, MimiConfig())
    B, frames = 4, 6
    orc.streaming(B)
    lat = orc.encode_to_latent(scenarios.mimi_noise(B, frames, seed=5))
    codes_o, margins = orc.quantize(lat, return_margins=True)
    with gpu.streaming(B):
        codes_g = torch.empty(B, 8, frames, dtype=torch.int64, device="cuda")
        from moshi_b200 import _lib
        lat_d = lat.cuda().contiguous()
        _lib.check(gpu._lib.b200_mimi_quantize(gpu._h, _lib.ptr(lat_d), frames, _lib.ptr(codes_g)))
        lat_q = gpu.decode_latent(codes_o.cuda())
    bad, unexcused = rvq_mismatches(codes_g, codes_o, margins, tol=1e-5)
    print(f"rvq on oracle latent: {bad} mismatches / {codes_o.numel()}, {unexcused} unexcused; "
          f"min margin {margins.min().item():.2e}")
    assert unexcused == 0 and bad <= 2
    torch.testing.assert_close(lat_q.cpu(), orc.dequantize(codes_o), rtol=1e-5, atol=1e-5)


@torch.no_grad()
def test_golden_sine_roundtrip(gpu, sd, golden_dir):
    """BASELINE.json configs[0]: 1 s 440 Hz sine, B=1; codes exact (margin-aware), PCM within tolerance."""
    gold = load_file(golden_dir / "mimi_sine.safetensors")
    cfg = MimiConfig()
    orc = MimiOracle(sd, cfg)
    orc.streaming(1)
    sine = scenarios.sine_1s()
    codes, pcm, margins = [], [], []
    with gpu.streaming(1):
        for f in range(12):
            x = sine[..., f * 1920:(f + 1) * 1920]
            _, m = orc.quantize(orc.encode_to_latent(x), return_margins=True)
            margins.append(m)
            c = gpu.encode(x.cuda())
            assert c.dtype == torch.int64 and c.shape == (1, 8, 1)
            codes.append(c)
            pcm.append(gpu.decode(gold["codes_stream"][..., f:f + 1].cuda()))
    codes, pcm, margins = torch.cat(codes, -1), torch.cat(pcm, -1), torch.cat(margins, -1)
    bad, unexcused = rvq_mismatches(codes, gold["codes_stream"], margins)
    print(f"sine: {bad} code mismatches of {codes.numel()} ({unexcused} unexcused); {stats('pcm', pcm, gold['pcm_stream'])}")
    assert unexcused == 0 and bad <= 2
    torch.testing.assert_close(pcm.cpu(), gold["pcm_stream"], rtol=0, atol=PCM_ATOL)
    # non-streaming API call: pads to 13 frames like the reference (compression.py:358)
    cb = gpu.encode(scenarios.sine_1s_full().cuda())
    assert cb.shape == (1, 8, 13)
    bad, unexcused = rvq_mismatches(cb[..., :12], gold["codes_batch"][..., :12], margins)
    assert unexcused == 0
    pb = gpu.decode(gold["codes_batch"].cuda())
    assert pb.shape == (1, 1, 13 * 1920)
    torch.testing.assert_close(pb.cpu(), gold["pcm_batch"], rtol=0, atol=PCM_ATOL)


@torch.no_grad()
def test_golden_masked_rows_and_reset(gpu, sd, golden_dir):
    """exec_mask pauses a row without touching its state; reset_streaming(mask) recycles a row."""
    gold = load_file(golden_dir / "mimi_masked.safetensors")
    B, frames = scenarios.MIMI_MASK_B, scenarios.MIMI_MASK_FRAMES
    pcm = scenarios.mimi_noise(B, frames)
    orc = MimiOracle(sd, MimiConfig())
    orc.streaming(B)
    total_bad = 0
    with gpu.streaming(B):
        for f in range(frames):
            scenarios.mimi_mask_events(gpu, f, B)
            scenarios.mimi_mask_events(orc, f, B)
            x = pcm[..., f * 1920:(f + 1) * 1920]
            _, margins = orc.quantize(orc.encode_to_latent(x), return_margins=True)
            live = orc.exec_mask.clone()
            c = gpu.encode(x.cuda())
            out = gpu.decode(gold["codes"][f].cuda())
            bad, unexcused = rvq_mismatches(c[live], gold["codes"][f][live], margins[live])
            total_bad += bad
            assert unexcused == 0, (f, bad)
            torch.testing.assert_close(out.cpu()[live], gold["pcm"][f][live], rtol=0, atol=PCM_ATOL, msg=f"frame {f}")
            orc.decode(gold["codes"][f])
    assert total_bad <= 3


@torch.no_grad()
def test_long_stream_ten_thousand_frames(gpu, sd):
    """40 sessions x 260 frames = 10 400 session-frames of streaming encode + decode beside the oracle (VERDICT r1 item 2: the
    3xTF32 tensor-core path must keep the RVQ indices exact over long streams): every code compared margin-aware (zero
    unexcused flips), PCM within tolerance on every frame, and the 250-slot rings of both bottleneck transformers wrap on
    the way (frames 250..259 overwrite the oldest keys)."""
    cfg = MimiConfig()
    B, frames = 40, 260
    pcm = scenarios.mimi_noise(B, frames, seed=77)
    orc = MimiOracle(sd, cfg)
    orc.streaming(B)
    bad = unexcused = total = 0
    worst_pcm = 0.0
    with gpu.streaming(B):
        for f in range(frames):
            x = pcm[..., f * 1920:(f + 1) * 1920]
            want, margins = orc.quantize(orc.encode_to_latent(x), return_margins=True)
            got = gpu.encode(x.cuda())
            b_, u_ = rvq_mismatches(got, want, margins)
            bad, unexcused, total = bad + b_, unexcused + u_, total + want.numel()
            out = gpu.decode(want.cuda()).cpu()          # both decoders are fed the oracle's codes: their states stay comparable
            worst_pcm = max(worst_pcm, (out - orc.decode(want)).abs().max().item())
    print(f"long stream: {bad} code mismatches of {total} ({unexcused} unexcused) over {B * frames} session-frames; worst PCM |d| {worst_pcm:.2e}")
    assert unexcused == 0 and bad <= total // 2000
    assert worst_pcm <= PCM_ATOL


def test_partial_frames_are_rejected(gpu):
    with gpu.streaming(1):
        with pytest.raises(RuntimeError):
            gpu.encode(torch.zeros(1, 1, 1000, device="cuda"))
        with pytest.raises(AssertionError):
            gpu.encode(torch.zeros(2, 1, 1920, device="cuda"))
    with pytest.raises(AssertionError):
        with gpu.streaming(1), gpu.streaming(1):
            pass
    gpu._stop()


@torch.no_grad()
def test_rows_are_independent_and_multiframe_equals_stepwise(gpu):
    """Size-independent properties at a serving-size batch: (1) a session's codes/PCM do not depend on
    which other sessions share the batch, (2) one call with n frames == n one-frame calls,
    (3) decode(encode(x)) state carries across calls (streaming == batch on the same signal)."""
    B, frames = 64, 4
    pcm = scenarios.mimi_noise(B, frames, seed=21).cuda()
    with gpu.streaming(B):
        codes_all = gpu.encode(pcm)
        out_all = gpu.decode(codes_all)
    with gpu.streaming(B):
        cs = [gpu.encode(pcm[..., f * 1920:(f + 1) * 1920]) for f in range(frames)]
        os_ = [gpu.decode(c) for c in cs]
    assert torch.equal(torch.cat(cs, -1), codes_all)
    assert torch.equal(torch.cat(os_, -1), out_all)
    with gpu.streaming(3):
        c3 = gpu.encode(pcm[5:8])
        o3 = gpu.decode(c3)
    assert torch.equal(c3, codes_all[5:8])
    # another batch size = another tiling / split-K of the tensor-core GEMMs, i.e. another fp32 summation order (measured 1.5e-5)
    torch.testing.assert_close(o3, out_all[5:8], rtol=0, atol=5e-5)
    assert codes_all.min() >= 0 and codes_all.max() < 2048 and codes_all.unique().numel() > 500


@torch.no_grad()
def test_host_buffer_entry_points(gpu):
    B = 4
    pcm = scenarios.mimi_noise(B, 1, seed=3)
    with gpu.streaming(B):
        want = gpu.encode(pcm.cuda())
        want_pcm = gpu.decode(want)
    with gpu.streaming(B):
        codes = torch.empty(B, 8, 1, dtype=torch.int64)
        gpu.encode_host(pcm.contiguous(), codes)
        out = torch.empty(B, 1, 1920)
        gpu.decode_host(codes, out)
    assert torch.equal(codes, want.cpu())
    assert torch.equal(out, want_pcm.cpu())


@torch.no_grad()
def test_graph_replay_equals_eager_launches(gpu):
    """One-frame encode / decode replayed as CUDA graphs == the same kernels launched one by one, bit for bit,
    including a paused row (exec_mask) and a recycled row (reset) in the middle of the stream."""
    B, frames = 5, 9
    pcm = scenarios.mimi_noise(B, frames, seed=23).cuda()

    def run(use_graph):
        gpu.use_graph = use_graph
        codes, outs = [], []
        with gpu.streaming(B):
            for f in range(frames):
                scenarios.mimi_mask_events(gpu, f, B)
                c = gpu.encode(pcm[..., f * 1920:(f + 1) * 1920])
                codes.append(c.cpu())
                outs.append(gpu.decode(c).cpu())
        gpu.use_graph = True
        return torch.cat(codes, -1), torch.cat(outs, -1)

    c_eager, p_eager = run(False)
    c_graph, p_graph = run(True)
    assert torch.equal(c_eager, c_graph)
    assert torch.equal(p_eager, p_graph)


@torch.no_grad()
def test_graph_replay_after_multiframe_quantize(gpu):
    """A multi-frame quantize between encodes (encode_to_latent(quantize=True)) leaves the captured encode graph valid:
    encode, quantize four frames at once, encode again, with graphs on == with graphs off, bit for bit at every call."""
    B = 3
    pcm = scenarios.mimi_noise(B, 7, seed=31).cuda()

    def run(use_graph):
        gpu.use_graph = use_graph
        with gpu.streaming(B):
            first = gpu.encode(pcm[..., :1920]).cpu()
            latent = gpu.encode_to_latent(pcm[..., 1920:5 * 1920], quantize=True).cpu()
            again = gpu.encode(pcm[..., 5 * 1920:]).cpu()
        gpu.use_graph = True
        return first, latent, again

    eager, graph = run(False), run(True)
    for want, got in zip(eager, graph):
        assert torch.equal(want, got)


@torch.no_grad()
def test_streaming_state_snapshot_roundtrip(gpu):
    """get_streaming_state / set_streaming_state (streaming.py:158-181): replaying from a snapshot reproduces the
    continuation bit for bit (conv carries, overlap-add partials, KV rings, offsets, masks all restored)."""
    B = 3
    pcm = scenarios.mimi_noise(B, 6, seed=5).cuda()
    with gpu.streaming(B):
        for f in range(3):
            gpu.decode(gpu.encode(pcm[..., f * 1920:(f + 1) * 1920]))
        snap = gpu.get_streaming_state()

        def tail():
            out = []
            for f in range(3, 6):
                c = gpu.encode(pcm[..., f * 1920:(f + 1) * 1920])
                out.append((c.cpu(), gpu.decode(c).cpu()))
            return out
        first = tail()
        gpu.set_streaming_state(snap)
        second = tail()
    for (c1, p1), (c2, p2) in zip(first, second):
        assert torch.equal(c1, c2) and torch.equal(p1, p2)
