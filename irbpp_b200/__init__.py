"""irbpp_b200: H100-native (sm_90a) packing-environment hot path of IR-BPP.

Submodules (imported lazily so CPU-only tooling can use ``shapes`` without the
CUDA library): ``shapes`` (shape tables), ``_lib`` (ctypes binding of the C-ABI
in ``include/irbpp.h``), ``vec_env`` (the reference's VecEnv surface on the GPU),
``envs`` (``make_vec_envs`` mirror), ``sharding`` (multi-GPU)."""
__version__ = "0.1.0"
# Stamp of the CUDA kernels' generation; bench.py only reports ncu DRAM traffic captured for this stamp.
KERNEL_VERSION = "r03-v29"
