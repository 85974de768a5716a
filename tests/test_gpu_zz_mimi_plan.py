"""GPU: the plan describes what runs.  At the first batch of every run of Mimi's per-frame kernel counts (b200_op_mimi_plan at this
device's SM count over 1..512 sessions), one encode and one decode frame advance b200_launch_count by exactly the plan's counts,
run eagerly (graphs off) and as a captured graph (a replay counts the kernels it holds)."""
import sys
from pathlib import Path

import pytest
import torch

from moshi_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def setup():
    sys.path.insert(0, str(ROOT / "tools"))
    import gen_mimi_plans as gen
    from moshi_b200.config import MimiConfig
    from moshi_b200.models import MimiModel
    from moshi_b200.synth import synth_mimi_state_dict
    cfg = MimiConfig()
    mimi = MimiModel(cfg, synth_mimi_state_dict(cfg, seed=7), device="cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    starts, last = [], None
    for B in range(1, gen.MAX_B + 1):
        rc, head, _ = gen.plan(B, sms)
        assert rc == _lib.B200_OK, B
        counts = (head["enc_launches"], head["dec_launches"])
        if counts != last:
            starts.append((B, counts))
            last = counts
    return gen, mimi, sms, starts


def _count(fn) -> int:
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.b200_launch_count()
    fn()
    torch.cuda.synchronize()
    return lib.b200_launch_count() - before


@pytest.mark.parametrize("graph", [False, True])
def test_frame_launches_match_plan(setup, graph):
    gen, mimi, sms, starts = setup
    assert len(starts) >= 2
    g = torch.Generator().manual_seed(0)
    for B, (enc, dec) in starts:
        pcm = (0.1 * torch.randn(B, 1, mimi.frame_size, generator=g)).cuda()
        mimi.use_graph = graph
        with mimi.streaming(B), torch.no_grad():
            codes = torch.empty(0)

            def encode():
                nonlocal codes
                codes = mimi.encode(pcm)

            got_enc = _count(encode)
            got_dec = _count(lambda: mimi.decode(codes))
        assert (got_enc, got_dec) == (enc, dec), (B, graph, sms)
    mimi.use_graph = True
