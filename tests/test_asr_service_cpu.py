"""CPU: the batched speech-to-text service's host side: the drop-in script's ``Config`` and the C ABI's declarations."""
import dataclasses
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

# rust/moshi-server/batched_asr.py:32-46, in declaration order
REFERENCE_CONFIG = {
    "log_folder": Path.home() / "tmp/tts-service",
    "hf_repo": "kyutai/moshiko-pytorch-bf16",
    "mimi_weight": None,
    "moshi_weight": Path.home() / "models/moshi/moshi_b1d046da_445/checkpoint.safetensors",
    "config_path": Path.home() / "models/moshi/moshi_b1d046da_445/config.json",
    "tokenizer": Path.home() / "models/mimi/tokenizer-e351c8d8-checkpoint125.safetensors",
    "asr_delay_in_tokens": 32,
    "device": "cuda",
    "temp": 0.0,
    "debug": False,
}


def test_config_has_the_reference_fields_and_defaults():
    from moshi_b200.batched_asr import Config
    assert [f.name for f in dataclasses.fields(Config)] == list(REFERENCE_CONFIG)
    cfg = Config()
    for name, want in REFERENCE_CONFIG.items():
        assert getattr(cfg, name) == want, name
    assert Config.from_dict({}) == cfg


def test_config_ignores_unknown_keys_and_reads_paths_from_strings(tmp_path):
    from moshi_b200.batched_asr import Config
    cfg = Config.from_dict({"log_folder": str(tmp_path / "logs"), "moshi_weight": "/m/w.safetensors", "asr_delay_in_tokens": 6,
                            "temp": 0, "batch_size": 64, "text_tokenizer_file": "tok.model", "debug": True})
    assert cfg.log_folder == tmp_path / "logs" and isinstance(cfg.log_folder, Path)
    assert cfg.moshi_weight == Path("/m/w.safetensors")
    assert cfg.asr_delay_in_tokens == 6 and cfg.temp == 0.0 and isinstance(cfg.temp, float) and cfg.debug is True
    assert cfg.mimi_weight is None and cfg.device == "cuda"


def test_asr_entry_points_are_declared_and_bound():
    from moshi_b200 import _lib, serving
    text = (ROOT / "include" / "moshi_b200.h").read_text()
    for fn in ("b200_asr_create", "b200_asr_step", "b200_asr_read_buffer", "b200_asr_destroy"):
        assert re.search(rf"\bint {fn}\(", text), fn
        assert fn in _lib.EXPORTED_SYMBOLS, fn
    flags = dict(re.findall(r"#define B200_ASR_(\w+) (\d+)", text))
    assert flags == {"ACTIVE": "1", "MARKER_RECEIVED": "2", "IS_EOS": "4"}
    assert (serving.MASK_ACTIVE, serving.MASK_MARKER_RECEIVED, serving.MASK_IS_EOS) == (1, 2, 4)
