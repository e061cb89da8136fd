"""CPU oracle for the PerspectiveFields inference hot path.  TEST INFRASTRUCTURE ONLY.

This package is a plain PyTorch-CPU / numpy restatement of the reference algorithm
(``perspective2d.PerspectiveFields.inference{,_batch}``, reference file:line cited per function).
It exists so that the CUDA product path can be checked on a box where the reference is not
present.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it; the product package ``perspectivefields_b200`` never does
and fails loudly when its CUDA library is missing.

Pinning (SURVEY.md section 8c): the reference ships no tests or golden vectors for this path and its
trained checkpoints are not available offline.  The oracle is therefore pinned against OUTPUTS OF THE
REFERENCE ITSELF, run unmodified in the build container through ``oracle/ref_shim.py`` on seeded
synthetic checkpoints (``oracle/weights_gen.py``) -- fixtures under ``tests/golden/`` made by
``tests/golden/make_golden.py`` -- and the Pillow resampler restatement is pinned against Pillow
itself (present on both boxes).
"""
