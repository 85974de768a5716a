"""moshi_b200 — H100-native (sm_90a) streaming inference path for Mimi + the Moshi LM decode step.

Public surface mirrors the reference package on this path::

    from moshi_b200.models import loaders, MimiModel, LMGen, LMModel

All arithmetic runs in ``moshi_b200/_C/libmoshi_b200.so`` (built by ``python -m moshi_b200.build``).
"""
__version__ = "0.1.0"
