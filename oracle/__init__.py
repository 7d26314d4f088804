"""oracle/ -- CPU restatement of the reference's batched SDF query path.

THIS PACKAGE IS TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import it, and only as
the checker / the timed CPU arm.  Nothing under pytorch_volumetric_b200/
imports it; the product path raises if the CUDA library is missing.

Layout
  geom.c / _geom.py          closest-point + ray-count arithmetic (Embree's role)
  tp_open3d.py               the Open3D calls the reference makes
  tp_multidim_indexing.py    TorchMultidimView (voxel index arithmetic)
  tp_pytorch_kinematics.py   Transform3d + URDF serial-chain FK
  tp_arm_utils.py            handle_batch_input / ensure_tensor / rand
  port.py                    restatement of the reference's OWN code
                             (sdf.py, voxel.py, model_to_sdf.py, chamfer.py)
  shims/                     packages named like the four third-party
                             dependencies that re-export the tp_* modules, so
                             the UNMODIFIED reference source of a checkout
                             (PVB_REFERENCE_SRC) can be imported by
                             make_golden.py to pin port.py
  make_golden.py             writes tests/golden/*.npz with the real reference
                             code running over the shims

Parity status: the reference's own logic is PINNED (port.py is checked
against the reference source executed over the same shims, and against the
committed golden vectors).  The third-party arithmetic under it (Open3D /
Embree, multidim_indexing, pytorch_kinematics, arm_pytorch_utilities -- none
present in this image, none vendored, all unpinned in pyproject.toml:54-61) is
restated from their published behaviour: "parity unpinned" at that boundary.
"""
