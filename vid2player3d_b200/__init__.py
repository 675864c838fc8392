"""vid2player3d_b200 - H100-native rollout hot path behind the vid2player3d Task surface.

Package contents (only what the hot path needs; SURVEY.md 8):
  csrc/            CUDA kernels + C ABI (include/b200env.h)
  native.py        ctypes binding (no CPU fallback)
  model_compiler   MJCF/STL -> constant block;  assets/compiled/*.npz
  motion_lib       flat SoA MoCap buffer
  tasks/           Python host mirror of the reference Task / VecTask classes
  shim/isaacgym    Level-B import shim so the reference's config / run modules import unchanged
  dist             PPO gradient all-reduce (replaces the Horovod call sites)
"""
__all__ = ["abi", "native", "model_compiler", "motion_lib"]
