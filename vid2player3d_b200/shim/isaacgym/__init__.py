"""Level-B import shim for the closed-source `isaacgym` package (SURVEY.md §8b).

The reference task / config modules do `from isaacgym import gymapi, gymtorch, gymutil`
and `from isaacgym.torch_utils import *`.  Isaac Gym Preview 4 is a binary tarball that
is not installable here (and has no sm_90 kernels), so this package restates the small
pure-python surface those imports need.  Physics itself is NOT here: it lives in the
CUDA extension behind `vid2player3d_b200.native` (C-ABI in include/b200env.h).
"""
from . import gymapi, gymtorch, gymutil, torch_utils  # noqa: F401
