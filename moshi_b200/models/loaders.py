"""Model factories with the reference's signatures (``moshi/moshi/models/loaders.py:145-446``).

``get_mimi`` / ``get_moshi_lm`` / ``CheckpointInfo`` accept what the reference accepts on this path
(safetensors checkpoints with the reference's key names, the JSON LM config, the nested Mimi config
dict) and return B200-backed ``MimiModel`` / ``LMModel`` objects.  With ``filename=None`` the
reference returns an un-initialised model; here that means seeded synthetic weights
(``moshi_b200.synth``), which is also what the tests and the bench use offline.
"""
from __future__ import annotations

import json
import typing as tp
from dataclasses import dataclass, field
from pathlib import Path

import torch

from ..config import LMConfig, MimiConfig
from ..synth import iter_synth_lm_tensors, synth_mimi_state_dict
from .compression import MimiModel
from .lm import LMModel

SAMPLE_RATE = 24000
FRAME_RATE = 12.5
TEXT_TOKENIZER_NAME = "tokenizer_spm_32k_3.model"
MOSHI_NAME = "model.safetensors"
MOSHI_Q8_NAME = "model.q8.safetensors"
MIMI_NAME = "tokenizer-e351c8d8-checkpoint125.safetensors"
DEFAULT_REPO = "kyutai/moshiko-pytorch-bf16"


def _is_safetensors(path: Path | str) -> bool:
    return Path(path).suffix in (".safetensors", ".sft", ".sfts")


def get_mimi(filename: str | Path | None, mimi_config: dict | None = None,
             device: torch.device | str = "cuda", num_codebooks: int = 8,
             synth_seed: int = 1234) -> MimiModel:
    """``loaders.get_mimi`` (loaders.py:323-363)."""
    cfg = MimiConfig.from_reference_dict(mimi_config, num_codebooks=num_codebooks)
    if filename is None:
        sd = synth_mimi_state_dict(cfg, seed=synth_seed)
    elif _is_safetensors(filename):
        from safetensors.torch import load_file
        sd = load_file(str(filename), device="cpu")
    else:
        sd = torch.load(filename, "cpu")["model"]
    model = MimiModel(cfg, sd, device=device)
    model.set_num_codebooks(num_codebooks)
    return model


def get_moshi_lm(filename: str | Path | None, lm_kwargs: dict | None = None,
                 device: torch.device | str = "cuda", dtype: torch.dtype = torch.bfloat16,
                 lora_weights: str | Path | None = None, fuse_lora: bool = False,
                 lm_kwargs_overrides: dict = {}, synth_seed: int = 4242,
                 synth_device: str | torch.device | None = None) -> LMModel:
    """``loaders.get_moshi_lm`` (loaders.py:366-446).  Checkpoints: ``model.safetensors`` (bf16), ``model.q8.safetensors``
    (loaders.py:33: every nn.Linear stored as a QLinear, ``weight`` int8 + ``weight_scb`` float32; needs ``quantize=True`` in the
    kwargs, like the reference), ``.gguf`` (the Rust stack's quantised form, F32 / F16 / BF16 / Q8_0 tensors under candle's names:
    ``moshi_b200/models/gguf.py``) and legacy ``.pt`` packages; packed ``in_proj_weight`` names are split (transformer.py:422-446).
    LoRA adapters are fused offline (loaders.py:512-513)."""
    if lora_weights is not None:
        raise ValueError("LoRA checkpoints are fused offline (loaders.py:512-513); pass fused weights")
    kwargs = dict(LMConfig().to_reference_kwargs() if lm_kwargs is None else lm_kwargs)
    kwargs.update(lm_kwargs_overrides)
    for k in ("lora", "lora_rank", "lora_scaling"):
        kwargs.pop(k, None)
    cfg = LMConfig.from_dict(kwargs)
    if filename is None:
        tensors: tp.Any = iter_synth_lm_tensors(cfg, seed=synth_seed, device=synth_device or "cpu", dtype=dtype)
    elif _is_safetensors(filename):
        from safetensors import safe_open

        def _stream():
            with safe_open(str(filename), framework="pt", device="cpu") as f:
                for key in f.keys():
                    yield key, f.get_tensor(key)
        tensors = _stream()
    elif Path(filename).suffix == ".gguf":
        # the Rust stack's quantised checkpoints (rust/moshi-core/src/nn.rs:9-116): candle tensor names, Q8_0 blocks dequantised
        if cfg.cross_attention:
            raise ValueError("GGUF checkpoints of a cross-attention LM are not supported; load its safetensors checkpoint")
        from .gguf import read_gguf
        _, tensors = read_gguf(filename)
    else:
        tensors = torch.load(filename, "cpu")["fsdp_best_state"]["model"]
    return LMModel(cfg, tensors, device=device, dtype=dtype)


@dataclass
class CheckpointInfo:
    """``loaders.CheckpointInfo`` (loaders.py:145-316) for local files; hub download needs a network."""
    moshi_weights: Path | None
    mimi_weights: Path | None
    tokenizer: Path | None
    lm_config: dict | None = None
    raw_config: dict | None = None
    mimi_config: dict | None = None
    model_type: str = "moshi"
    lora_weights: Path | None = None
    lm_gen_config: dict = field(default_factory=dict)
    tts_config: dict = field(default_factory=dict)
    stt_config: dict = field(default_factory=dict)
    model_id: dict = field(default_factory=dict)

    @staticmethod
    def from_hf_repo(hf_repo: str, moshi_weights=None, mimi_weights=None, tokenizer=None, config_path=None,
                     mimi_config_path=None, lora_weights=None, revision=None) -> "CheckpointInfo":
        from huggingface_hub import hf_hub_download

        def fetch(name_or_path, default_name):
            if name_or_path is not None:
                return Path(name_or_path)
            return Path(hf_hub_download(hf_repo, default_name, revision=revision))
        lm_config = raw = None
        names = {"moshi": MOSHI_NAME, "mimi": MIMI_NAME, "tok": TEXT_TOKENIZER_NAME}
        if config_path is None:
            try:
                config_path = hf_hub_download(hf_repo, "config.json", revision=revision)
            except Exception:
                config_path = None
        gen_cfg: dict = {}
        if config_path is not None:
            raw = json.loads(Path(config_path).read_text())
            lm_config = dict(raw)
            names["moshi"] = lm_config.pop("moshi_name", MOSHI_NAME)
            names["mimi"] = lm_config.pop("mimi_name", MIMI_NAME)
            names["tok"] = lm_config.pop("tokenizer_name", TEXT_TOKENIZER_NAME)
            for k in ("mimi_config_name", "lora_name", "tts_config", "stt_config", "model_id"):
                lm_config.pop(k, None)
            lm_config.pop("model_type", None)
            gen_cfg = lm_config.pop("lm_gen_config", {})
        mimi_cfg = json.loads(Path(mimi_config_path).read_text()) if mimi_config_path else None
        return CheckpointInfo(fetch(moshi_weights, names["moshi"]), fetch(mimi_weights, names["mimi"]),
                              fetch(tokenizer, names["tok"]), lm_config, raw, mimi_cfg, lm_gen_config=gen_cfg)

    def get_mimi(self, device: torch.device | str = "cuda") -> MimiModel:
        if self.lm_config is None:
            num_codebooks = 8
        else:
            num_codebooks = max(self.lm_config["dep_q"], self.lm_config["n_q"] - self.lm_config["dep_q"])
        return get_mimi(self.mimi_weights, self.mimi_config, num_codebooks=num_codebooks, device=device)

    def get_moshi(self, device: torch.device | str = "cuda", dtype: torch.dtype = torch.bfloat16,
                  load_weight: bool = True, **kwargs) -> LMModel:
        return get_moshi_lm(self.moshi_weights if load_weight else None, lm_kwargs=self.lm_config,
                            device=device, dtype=dtype, **kwargs)

    def get_text_tokenizer(self):
        import sentencepiece
        return sentencepiece.SentencePieceProcessor(str(self.tokenizer))
