"""CPU oracle for the halo-exchange / jacobi3d hot path of cwpearson/stencil.

TEST INFRASTRUCTURE ONLY.  Nothing under ``stencil_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs use it, and only as the checker or
as the timed CPU baseline -- never as the thing shipped.

Three layers, each citing the reference file:line it restates:

* :mod:`oracle.geometry`   -- integer geometry, partition, planner (pure Python)
* :mod:`oracle.np_oracle`  -- pack / unpack / translate / exchange / jacobi in numpy
* :mod:`oracle.c_oracle`   -- the same data movement + jacobi in plain C (+OpenMP),
  ``oracle/stencil_oracle.c``; this is what the CPU baseline times.

Parity status: pinned.  The restatement is checked against every golden value
the reference's own tests hold for this path (``tests/test_oracle_golden.py``)
and against vectors dumped from the reference's own host code compiled here
(``oracle/ref/``, ``tests/golden/ref_geometry.json``).  Jacobi numerics have no
golden in the reference (SURVEY.md 8c: "parity unpinned" for jacobi values);
there the two independent restatements (numpy, C) are cross-checked bit-exactly
and the reference's own ``stencil_kernel`` is run beside ours on the GPU
(``oracle/_ref``).
"""
