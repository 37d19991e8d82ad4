"""CPU oracle — TEST INFRASTRUCTURE ONLY.

A restatement, on the CPU, of the reference algorithms on the hot path
(llm-d/llm-d-kv-cache @ 82d31d1).  Nothing under ``oracle/`` is part of the
product: only ``tests/`` (the pytest suite and the two measurement / sanitizer
drivers kept there: ``bench_extras.py`` (part of bench.py), ``tests/bench_fused.py``, ``tests/bench_hash.py``, ``tests/sanitize_smoke.py``, ``tests/soak_engine.py``, ``tests/soak_hash.py``),
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it, and only as the checker / the reported
baseline.  ``tools/`` never does.  The product (``llm-d-kv-cache_b200``) never
imports this package and has no CPU fallback.

Parity status (see DESIGN.md "Oracle"):
  * kvblock hashing      — PINNED by the reference's golden vectors
                            (tests/golden/kvblock_golden.json, 1 + 104 keys).
  * index / scorer       — pinned by the reference's known-answer tests
                            (scores 3.0 / 2.5 / 1.8 ..., transcribed in tests/).
  * offload staging/file — no golden bytes exist in the reference (layout is only
                            pinned by read-after-write symmetry); the layout is
                            restated from the code and cross-checked against files
                            the reference engine wrote (tests/golden/ref_offload_files.json).
"""
