"""leetcuda_b200 — H100-native (sm_90a) drop-in for LeetCUDA's two hot paths.

Sub-modules mirror the reference's extension modules one to one:

* :mod:`leetcuda_b200.hgemm`      — `toy_hgemm` / `hgemm_lib`  (kernels/hgemm/pybind/hgemm.cc)
* :mod:`leetcuda_b200.flash_attn` — `flash_attn_lib`           (kernels/flash-attn/pybind/flash_attn.cc)
* :mod:`leetcuda_b200.ffpa_attn`  — `ffpa_attn` / `pyffpa_cuda` (ffpa-attn/ffpa_attn/interface.py)

All compute happens in hand-written sm_90a kernels behind the C ABI of
include/leetcuda_b200.h (see :mod:`leetcuda_b200._capi`).
"""
__version__ = "0.1.0"
