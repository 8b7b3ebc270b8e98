"""Host-side Lie-group tensors over the lietorch_backends extension (SE3 / SO3).

Mirror of the reference's dpvo/lietorch package interface (groups.py:51-322, group_ops.py:7-102)
so DPVO-style code (`SE3(poses)[:, jj] * SE3(poses)[:, ii].inv()`, `.retr`, `.adjT`, `.matrix()`,
`lietorch.stack`) runs unchanged on top of the sm_90a kernels.
"""
from .groups import SO3, SE3, RxSO3, Sim3, LieGroup, LieGroupParameter, cat, stack  # noqa: F401
