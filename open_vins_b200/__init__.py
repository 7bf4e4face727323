"""open_vins_b200 — H100-native MSCKF update engine behind the OpenVINS State/Updater surfaces.

Only what the hot path needs lives here: csrc/ (sm_90a CUDA kernels + the C ABI of include/ovb200.h),
capi.py (ctypes view of that ABI), sim.py (rpng_sim-like synthetic update cases), build.py (nvcc build).
"""
__version__ = "0.1.0"
