"""CPU oracle for the ZhiLight quantized-decode hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` may be imported by the
product package ``zhilight_b200``; only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s cpu_baseline / ``--impl reference`` leg use it, and there only
as the checker / the reported CPU baseline.

Every function restates, in numpy, the algorithm of a reference file under
the reference checkout (cited per function as file:line).  Integer / byte stages
are exact; float stages are fp32 (optionally emulating the reference's fp16
partial sums).

Pinning status: the reference has no golden vectors for any quantized or
decode path (SURVEY.md section 8c).  The oracle is pinned against outputs of
the reference's own kernels compiled for sm_90a (``oracle/_ref``; fixtures in
``tests/golden/ref_*.npz`` produced by ``oracle/gen_ref_golden.py`` on a GPU
box).  Until those fixtures are committed the header of DESIGN.md says
"parity unpinned".
"""
