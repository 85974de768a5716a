"""The oracle's spec of an LM with a depformer weight-sharing schedule and / or low-rank depformer embeddings.

``oracle.lm.LMSpec.from_config`` restates the 7B family, whose spec leaves both at their defaults; the oracle itself steps
both options (``oracle/lm.py``: ``depformer_schedule`` in forward_depformer and the transformer, the ``low_rank`` linear in
scaled_embedding), so the spec of such a configuration is the family's spec with the two fields set."""
from __future__ import annotations

import dataclasses

from oracle.lm import LMSpec


def sched_spec(cfg) -> LMSpec:
    s = cfg.depformer_weights_per_step_schedule
    return dataclasses.replace(LMSpec.from_config(cfg), depformer_schedule=None if s is None else list(s),
                               depformer_low_rank=cfg.depformer_low_rank_embeddings)
