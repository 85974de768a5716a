"""CPU: depformer weight-sharing schedules and low-rank depformer embeddings (lm.py:125-127, 172-196; transformer.py:291-316,
399-401; lm_utils.py:80-124).  The configuration's refusals, its round trip to the reference's keyword arguments, the synthetic
checkpoint's names and shapes, the two C setters' argument checks (no GPU needed), and the oracle against the reference-recorded
fixture tests/golden/lm_tiny_sched.* (tools/gen_golden_sched.py), bit for bit."""
import ctypes as C
import dataclasses
import json

import pytest
import torch
from safetensors.torch import load_file

from moshi_b200.config import LMConfig, tiny_lm_config
from moshi_b200.synth import lm_tensor_specs, synth_lm_state_dict
from oracle import scenarios
from oracle.lm import LMOracle
from tests.depformer_sched import sched_spec

SCHEDULE = [0, 1, 2, 2, 2, 3, 3, 3]


@pytest.mark.parametrize("over,needle", [
    (dict(depformer_weights_per_step_schedule=SCHEDULE, depformer_multi_linear=False), "without depformer_multi_linear"),
    (dict(depformer_weights_per_step_schedule=SCHEDULE, depformer_weights_per_step=False), "without depformer_multi_linear"),
    (dict(depformer_weights_per_step_schedule=[0, 1, 2]), "of length 3"),
    (dict(depformer_weights_per_step_schedule=[0, 1, 2, 2, 2, 3, 3, 8]), "entries must be in [0, dep_q = 8)"),
    (dict(depformer_weights_per_step_schedule=[0, 1, 2, 2, 2, 3, 3, -1]), "entries must be in [0, dep_q = 8)"),
    (dict(depformer_low_rank_embeddings=0), "the rank must be in [1, 4096]"),
    (dict(depformer_low_rank_embeddings=4097), "the rank must be in [1, 4096]"),
])
def test_unsupported_schedules_and_ranks_are_refused(over, needle):
    cfg = tiny_lm_config(**over)
    with pytest.raises(ValueError) as e:
        cfg.check_supported()
    assert needle in str(e.value)
    d = {k: v for k, v in dataclasses.asdict(cfg).items()}
    with pytest.raises(ValueError):
        LMConfig.from_dict(d)


def test_supported_options_round_trip_to_the_reference_kwargs():
    cfg = LMConfig.from_dict({**dataclasses.asdict(tiny_lm_config()), "depformer_weights_per_step_schedule": SCHEDULE,
                              "depformer_low_rank_embeddings": 32})
    kw = cfg.to_reference_kwargs()
    assert kw["depformer_weights_per_step_schedule"] == SCHEDULE and kw["depformer_low_rank_embeddings"] == 32
    assert LMConfig.from_dict({**kw, "conditioners": None, "fuser": None}) == cfg
    assert cfg.depformer_n_sets == 4 and tiny_lm_config().depformer_n_sets == 8
    plain = tiny_lm_config().to_reference_kwargs()
    assert plain["depformer_weights_per_step_schedule"] is None and plain["depformer_low_rank_embeddings"] is None


def test_synthetic_checkpoint_has_the_reference_names_and_shapes():
    """n_sets = max(schedule) + 1 depformer_in linears and weight sets per layer (lm.py:177-178, transformer.py:399-401), and
    [V, r] tables with a [dd, r] low_rank linear each (lm_utils.py:80-94).  Unscheduled full-rank specs are unchanged."""
    cfg = tiny_lm_config(depformer_weights_per_step_schedule=SCHEDULE, depformer_low_rank_embeddings=32)
    specs = {k: s for k, s, _ in lm_tensor_specs(cfg)}
    dd = cfg.depformer_dim
    assert sorted(k for k in specs if k.startswith("depformer_in.")) == [f"depformer_in.{j}.weight" for j in range(4)]
    assert {k.split(".")[5] for k in specs if ".self_attn.in_projs." in k} == {"0", "1", "2", "3"}
    assert {k.split(".")[4] for k in specs if k.startswith("depformer.") and ".gating." in k} == {"0", "1", "2", "3"}
    assert specs["depformer_text_emb.weight"] == (cfg.text_card + 1, 32)
    assert specs["depformer_text_emb.low_rank.weight"] == (dd, 32)
    assert specs["depformer_emb.6.weight"] == (cfg.card + 1, 32) and specs["depformer_emb.6.low_rank.weight"] == (dd, 32)
    assert [k for k, _, _ in lm_tensor_specs(tiny_lm_config())] == \
        [k for k, _, _ in lm_tensor_specs(tiny_lm_config(depformer_weights_per_step_schedule=list(range(8))))]


def test_candle_layout_is_refused_for_scheduled_and_low_rank_models():
    """The candle layout (scripts/import_rust.py:69-110) stores one slice per depformer step, a schedule unrolled: slice k holds
    set schedule[k].  Renamed to set k, a scheduled model would read set 2's weights for set 3 under [0, 1, 2, 2, 2, 3, 3, 3],
    so such checkpoints are refused, as are candle-layout low-rank tables; the other layouts and models are unaffected."""
    from moshi_b200.models.state_dict import candle_refusal, normalize_lm_state_dict
    sched = tiny_lm_config(depformer_weights_per_step_schedule=SCHEDULE)
    low = tiny_lm_config(depformer_low_rank_embeddings=32)
    plain = tiny_lm_config()
    for key in ("depformer.3.linear_in.weight", "depformer.5.transformer.layers.0.gating.linear_in.weight",
                "depformer.1.emb.low_rank.weight"):
        assert "depformer_weights_per_step_schedule" in candle_refusal(sched, key)
        assert "depformer_low_rank_embeddings" in candle_refusal(low, key)
        assert candle_refusal(plain, key) is None
    for cfg in (sched, low, plain):
        assert candle_refusal(cfg, "depformer_in.3.weight") is None
        assert candle_refusal(cfg, "depformer.layers.0.gating.3.linear_in.weight") is None
    # what the refusal prevents: the unrolled slice of step 5 lands on set 5, which the schedule never reads
    t = torch.zeros(1)
    assert "depformer_in.5.weight" in normalize_lm_state_dict({"depformer.5.linear_in.weight": t})


@pytest.fixture(scope="module")
def lib():
    from moshi_b200 import _lib
    from moshi_b200.build import build
    build()
    return _lib


def _handle(_lib, cfg: LMConfig) -> C.c_void_p:
    from moshi_b200.models.lm import _config_struct
    h = C.c_void_p()
    _lib.check(_lib.lib().b200_lm_create(C.byref(_config_struct(cfg)), C.byref(h)))
    return h


def test_setters_check_their_arguments_without_a_gpu(lib):
    L = lib.lib()
    h = _handle(lib, tiny_lm_config())
    try:
        def sched(vals, n=None):
            arr = (C.c_int * max(len(vals), 1))(*vals)
            return L.b200_lm_set_depformer_schedule(h, arr, len(vals) if n is None else n)
        assert sched(SCHEDULE) == lib.B200_OK
        assert sched([]) == lib.B200_OK                              # back to one set per sub-step
        assert sched(SCHEDULE[:7]) == lib.B200_ERR_INVALID
        assert b"8 steps" in L.b200_last_error()
        assert sched(SCHEDULE + [0]) == lib.B200_ERR_INVALID
        assert sched([0, 1, 2, 2, 2, 3, 3, 8]) == lib.B200_ERR_INVALID
        assert b"outside [0, 8)" in L.b200_last_error()
        assert sched([0, 1, 2, 2, 2, 3, 3, -1]) == lib.B200_ERR_INVALID
        assert L.b200_lm_set_depformer_schedule(h, None, 8) == lib.B200_ERR_INVALID
        assert L.b200_lm_set_depformer_schedule(None, None, 0) == lib.B200_ERR_INVALID
        for r, rc in ((32, lib.B200_OK), (0, lib.B200_OK), (4096, lib.B200_OK), (-1, lib.B200_ERR_INVALID),
                      (4097, lib.B200_ERR_INVALID)):
            assert L.b200_lm_set_depformer_low_rank(h, r) == rc, r
        assert L.b200_lm_set_depformer_low_rank(None, 8) == lib.B200_ERR_INVALID
    finally:
        L.b200_lm_destroy(h)
    # a model without a depformer has no steps to schedule, and no tables to factor: the rank is ignored, as the reference does
    h = _handle(lib, dataclasses.replace(tiny_lm_config(), dep_q=0, delays=[0] * 17))
    try:
        assert L.b200_lm_set_depformer_low_rank(h, 8) == lib.B200_OK
        assert L.b200_lm_set_depformer_schedule(h, (C.c_int * 1)(0), 1) == lib.B200_ERR_INVALID
        assert L.b200_lm_set_depformer_schedule(h, None, 0) == lib.B200_OK
    finally:
        L.b200_lm_destroy(h)


@pytest.mark.parametrize("run,sampling", [("greedy", False), ("sampled", True)])
def test_oracle_reproduces_the_reference_fixture(golden_dir, run, sampling):
    info = json.loads((golden_dir / "lm_tiny_sched.json").read_text())
    assert info["runs"][run]["oracle_bit_exact_tokens"] and info["runs"][run]["oracle_bit_exact_text_logits"]
    gold = load_file(golden_dir / "lm_tiny_sched.safetensors")
    cfg = tiny_lm_config(depformer_weights_per_step_schedule=info["schedule"], depformer_low_rank_embeddings=info["low_rank"])
    sd = synth_lm_state_dict(cfg, seed=info["seed"])
    B, steps = info["B"], info["steps"]
    codes = gold["codes"]
    assert torch.equal(codes, scenarios.lm_input_codes(cfg, B, steps, seed=info["seed"]))
    orc = LMOracle(sd, sched_spec(cfg), use_sampling=sampling)
    orc.streaming(B)
    torch.manual_seed(info["noise_seed"])
    for i in range(steps):
        scenarios.lm_mask_events(orc, i, B)
        nt, na = scenarios.lm_noise(cfg, B) if sampling else (None, None)
        dbg: dict = {}
        o = orc.step(codes[i], nt, na, debug=dbg)
        assert torch.equal(dbg["text_logits"][:, 0, 0], gold[f"{run}.text_logits"][i]), i
        want = gold[f"{run}.tokens"][i]
        if o is None:
            assert bool((want == info["none_marker"]).all()), i
        else:
            assert torch.equal(o, want), i
