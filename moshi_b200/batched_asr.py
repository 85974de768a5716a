"""Drop-in for ``rust/moshi-server/batched_asr.py``: the script the Rust server's batched speech-to-text module loads
(``py_basr_module.rs``: ``PyModule::from_code(script).getattr("init").call1((batch_size, config))``) and then drives with
``step(batch_pcm, flags_out, tokens_out, extra_heads, updates)`` every 80 ms.

Point the module's ``script`` setting at this file.  The server loads it as a standalone module, so everything below is
imported by absolute name: ``moshi_b200`` must be importable by the server's Python.  The returned service is
``moshi_b200.serving.ASRService``, which runs each frame as one device chain with a single host wait.
"""
import dataclasses
from dataclasses import dataclass
from pathlib import Path

import torch

from moshi_b200.models import loaders
from moshi_b200.serving import ASRService


@dataclass
class Config:
    """The reference's ``Config`` (batched_asr.py:32-46): same field names and defaults.  ``from_dict`` ignores unknown keys
    and turns strings into paths, as the reference's pydantic model does."""
    log_folder: Path = Path.home() / "tmp/tts-service"
    hf_repo: str = loaders.DEFAULT_REPO
    mimi_weight: Path | None = None
    moshi_weight: Path = Path.home() / "models/moshi/moshi_b1d046da_445/checkpoint.safetensors"
    config_path: Path = Path.home() / "models/moshi/moshi_b1d046da_445/config.json"
    tokenizer: Path = Path.home() / "models/mimi/tokenizer-e351c8d8-checkpoint125.safetensors"
    asr_delay_in_tokens: int = 32
    device: str = "cuda"
    temp: float = 0.0
    debug: bool = False

    @classmethod
    def from_dict(cls, values: dict) -> "Config":
        known = {f.name for f in dataclasses.fields(cls)}
        cfg = cls(**{k: v for k, v in values.items() if k in known})
        for name in ("log_folder", "mimi_weight", "moshi_weight", "config_path", "tokenizer"):
            v = getattr(cfg, name)
            if v is not None:
                setattr(cfg, name, Path(v))
        cfg.asr_delay_in_tokens = int(cfg.asr_delay_in_tokens)
        cfg.temp = float(cfg.temp)
        cfg.debug = bool(cfg.debug)
        return cfg


def init(batch_size: int, config_override: dict) -> ASRService:
    """batched_asr.py:49-82: loads Mimi (with ``max(dep_q, n_q - dep_q)`` codebooks) and the LM, and builds the service."""
    config = Config.from_dict(dict(config_override))
    config.log_folder.mkdir(parents=True, exist_ok=True)

    print("retrieving checkpoint...")
    checkpoint_info = loaders.CheckpointInfo.from_hf_repo(
        config.hf_repo,
        moshi_weights=config.moshi_weight,
        mimi_weights=config.mimi_weight,
        config_path=config.config_path,
        tokenizer=config.tokenizer,
    )
    print("done.")
    print("loading mimi...")
    mimi = checkpoint_info.get_mimi(device=config.device)
    print("mimi loaded.")
    print("loading moshi...")
    lm = checkpoint_info.get_moshi(device=config.device, dtype=torch.bfloat16)
    print("moshi loaded.")
    print("warming up...")
    service = ASRService(batch_size, lm, mimi, asr_delay_in_tokens=config.asr_delay_in_tokens, temp=config.temp)
    print("ready to roll !")
    return service
