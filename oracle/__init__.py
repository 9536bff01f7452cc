"""CPU oracle for the EmerNeRF per-ray-batch hot path.  TEST INFRASTRUCTURE ONLY.

Nothing under ``emernerf_b200/`` may import this package.  The only legal
importers are ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` -- and there only as the *checker*
(or the timed CPU baseline), never as the product path.

What is restated here and how it is pinned
------------------------------------------
* ``oracle.hotpath`` restates the reference's **in-tree Python** for the path
  (``radiance_fields/{radiance_field,render_utils,encodings,mlp,nerf_utils}.py``
  and ``third_party/nerfacc_prop_net.py`` at NVlabs/EmerNeRF@8c051d7) as plain
  functions over a state-dict.  It is PINNED: ``tests/golden/make_golden.py``
  imports the reference's own modules from a checkout (``EMER_REFERENCE_ROOT``; with the three
  stand-in modules of ``oracle.ref_shims`` injected), runs them, and commits the
  results under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this
  restatement against those vectors.

* ``oracle.tcnn_ref`` restates tiny-cuda-nn's ``HashGrid`` encoding
  (``include/tiny-cuda-nn/encodings/grid.h``; tiny-cuda-nn is installed
  *unpinned from master* by the reference, README.md:51) and
  ``oracle.nerfacc_ref`` restates the seven nerfacc symbols the path uses
  (nerfacc pinned at 8340e19daad4bafe24125150a8c56161838086fa, README.md:50).
  Neither library's source is in the reference tree, and neither is
  installed in the build environment.  **Parity unpinned** for these two: the only published
  known-answer vector available offline is the ``importance_sampling``
  docstring example of nerfacc (checked in ``tests/test_oracle_nerfacc.py``);
  everything else is anchored on the reference's call sites.
"""
