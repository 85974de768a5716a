"""CPU oracle for the Mimi + Moshi-LM streaming hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``moshi_b200/`` imports this package; it is used by
``tests/``, by ``__graft_entry__.smoke()`` as the checker, and by ``bench.py`` for the
``cpu_baseline`` / ``--impl reference`` timing leg.

The oracle restates, as plain functional PyTorch-on-CPU code with explicit state, the algorithms of
the reference's PyTorch path (each function cites the reference ``file:line`` it follows).  It is
pinned against the unmodified reference by ``oracle/gen_golden.py`` (run in the build container,
where ``$MOSHI_REFERENCE`` exists) — see ``tests/golden/MANIFEST.json`` for what was compared and the
fixtures that travel to the GPU box.
"""
