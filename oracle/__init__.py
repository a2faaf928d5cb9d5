"""oracle/ -- TEST INFRASTRUCTURE ONLY (CPU restatement of the reference's sampling hot path).

Nothing in the product package (`targetdiff_b200/`) may import from here.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` / `--impl reference` legs use it, and
there only as the checker / the reported CPU baseline -- never as the thing measured or shipped.

Contents
--------
shims/      pure-torch stand-ins for the un-vendored third-party wheels the reference imports
            (torch_scatter 2.1.0, torch_geometric 2.2.0 `knn_graph`, easydict) so that the
            UNMODIFIED reference `models/*.py` can be imported from a reference checkout in the build
            container (never on the GPU box -- the reference tree does not travel).
restate.py  op-by-op CPU restatement of the path (every function cites the reference file:line).
synth.py    seeded synthetic pockets / weights / noise tapes shared by tests and bench.
refload.py  imports the reference under the shims (build container only).
make_golden.py  regenerates tests/golden/*.npz by running the reference itself.

Parity pinning
--------------
The reference ships no tests, golden vectors or checkpoints (SURVEY.md section 4).  The restatement
is pinned against the reference *itself*, executed here under the shims (tests/test_oracle_vs_reference.py,
bit-exact) and against committed golden vectors produced by that run (tests/golden/).
The arithmetic of the third-party kernels (torch_cluster knn tie-breaking / rounding, torch_scatter
reduction order) is NOT in the reference tree and nothing in the reference pins it:
**parity unpinned at that boundary** -- we fix canonical semantics (SURVEY.md Appendix A.3/A.4).
"""
