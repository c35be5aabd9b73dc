"""TEST INFRASTRUCTURE — build the UNMODIFIED reference kernels for sm_90a.

Compiles the reference's own CUDA sources *where they lie* in the reference checkout (/root/reference,
or $LEETCUDA_REFERENCE; nothing is copied) together with the small binding files in this
directory into python extension modules under oracle/_ref/ (git-ignored):

    oracle/_ref/ref_hgemm/ref_hgemm.so    kernels/hgemm       (all tensor-core ops + cuBLAS op)
    oracle/_ref/ref_fa/ref_fa.so          kernels/flash-attn  (split-q, share-qkv{,acc_f32,swizzle_qkv}, tiling-qkv)
    oracle/_ref/ref_ffpa/ref_ffpa.so      ffpa-attn           (ffpa_mma_acc_{f16,f32}_L1)
    oracle/_ref/ref_sgemm/ref_sgemm.so    kernels/sgemm       (TF32 wmma ops + cuBLAS ops)
    oracle/_ref/ref_merge/ref_merge.so    kernels/openai-triton/merge-attn-states (merge_attn_states_cuda)
    oracle/_ref/ref_rope/ref_rope.so      kernels/rope        (rope_f32, rope_f32_v2, rope_f32x4_pack)
    oracle/_ref/ref_rmsnorm/ref_rmsnorm.so kernels/rms-norm   (the nine rms_norm_* ops)

Flags follow the reference's JIT builds (kernels/hgemm/tools/utils.py:62-98,
kernels/flash-attn/flash_attn_mma.py:151-195, ffpa-attn/env.py:312-343, kernels/sgemm/sgemm.py:11-31) with the arch
set to sm_90a.  The modules are the on-box comparator and the source of the
golden vectors under tests/golden/ (oracle/gen_golden.py); the product never
loads them.

`scripts` stages the reference's own BENCH / TEST SCRIPTS (python files only, byte for byte) under
oracle/_ref/scripts/ in their original directory layout, so that a GPU machine without a reference
checkout can run them unmodified against the mirror (tools/run_reference_script.py,
tests/test_reference_scripts_gpu.py).  Like everything under oracle/_ref/ they are never committed.

    python oracle/build_ref.py [hgemm] [fa] [ffpa] [sgemm] [merge] [rope] [rmsnorm] [scripts]
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
OUT = HERE / "_ref"
# the reference checkout (xlite-dev/LeetCUDA) the comparators are built from; $LEETCUDA_REFERENCE overrides the default
REF = Path(os.environ.get("LEETCUDA_REFERENCE", "/root/reference"))


def reference_present() -> bool:
    try:
        return REF.is_dir()
    except OSError:   # e.g. a path under a directory this user may not enter
        return False

COMMON = [
    "-O3", "-std=c++17",
    "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
    "-U__CUDA_NO_HALF2_OPERATORS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
    "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math",
    "-diag-suppress", "177",
    "-gencode", "arch=compute_90a,code=sm_90a",
]


def _load(name, sources, cuda_flags, cflags=()):
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 8))
    from torch.utils.cpp_extension import load
    bdir = OUT / name
    bdir.mkdir(parents=True, exist_ok=True)
    return load(name=name, sources=[str(s) for s in sources], extra_cuda_cflags=list(cuda_flags),
                extra_cflags=["-std=c++17", *cflags], build_directory=str(bdir), verbose=True)


def build_hgemm():
    k = REF / "kernels" / "hgemm"
    srcs = [k / p for p in [
        "cublas/hgemm_cublas.cu", "wmma/hgemm_wmma_stage.cu", "mma/basic/hgemm_mma.cu",
        "mma/basic/hgemm_mma_stage.cu", "mma/basic/hgemm_mma_stage_tn.cu",
        "mma/swizzle/hgemm_mma_stage_swizzle.cu", "mma/swizzle/hgemm_mma_stage_tn_swizzle_x4.cu",
        "cutlass/hgemm_mma_stage_tn_cute.cu"]] + [HERE / "ref_glue_hgemm.cc"]
    flags = COMMON + ["-DNO_MMA_HGEMM_BIN", "-DNO_WMMA_HGEMM_BIN", "-DNO_CUTE_HGEMM_BIN",
                      "-DNO_CUBLAS_HGEMM_BIN", f"-I{k}", f"-I{k}/utils",
                      f"-I{REF}/third-party/cutlass/include",
                      f"-I{REF}/third-party/cutlass/tools/util/include", "-lcublas"]
    return _load("ref_hgemm", srcs, flags, cflags=[f"-I{HERE}"])


def build_fa():
    k = REF / "kernels" / "flash-attn"
    srcs = [k / p for p in [
        "mma/basic/flash_attn_mma_split_q.cu", "mma/basic/flash_attn_mma_share_qkv.cu",
        "mma/basic/flash_attn_mma_share_qkv_F32F16F16F32.cu", "mma/basic/flash_attn_mma_tiling_qkv.cu",
        "mma/swizzle/flash_attn_mma_share_qkv_swizzle_qkv.cu"]] + [HERE / "ref_glue_fa.cc"]
    flags = COMMON + [f"-I{k}", f"-I{k}/utils", f"-I{k}/mma", f"-I{k}/mma/basic",
                      f"-I{k}/mma/swizzle"]
    return _load("ref_fa", srcs, flags, cflags=[f"-I{HERE}"])


def build_ffpa():
    k = REF / "ffpa-attn"
    srcs = [k / "csrc/cuffpa/ffpa_attn_F16F16F16_L1.cu", k / "csrc/cuffpa/ffpa_attn_F16F16F32_L1.cu",
            HERE / "ref_glue_ffpa.cc"]
    flags = COMMON + ["-DENABLE_FFPA_ALL_STAGES", f"-I{k}/include", f"-I{k}/csrc/cuffpa"]
    return _load("ref_ffpa", srcs, flags, cflags=[f"-I{HERE}"])


def build_sgemm():
    k = REF / "kernels" / "sgemm"
    srcs = [k / "sgemm_wmma_tf32_stage.cu", k / "sgemm_cublas.cu", HERE / "ref_glue_sgemm.cc"]
    return _load("ref_sgemm", srcs, COMMON + ["-lcublas"], cflags=[f"-I{HERE}"])


def build_merge():
    # the file carries its own PYBIND11_MODULE; flags of cuda_merge_attn_states.py:8-19 (no fast-math)
    src = REF / "kernels" / "openai-triton" / "merge-attn-states" / "cuda_merge_attn_states.cu"
    flags = [f for f in COMMON if f != "--use_fast_math"]
    return _load("ref_merge", [src], flags)


def build_rope():
    # the file carries its own PYBIND11_MODULE; flags of kernels/rope/rope.py:10-24 (--use_fast_math included)
    return _load("ref_rope", [REF / "kernels" / "rope" / "rope.cu"], COMMON)


def build_rmsnorm():
    # own PYBIND11_MODULE; flags of kernels/rms-norm/rms_norm.py:10-24
    return _load("ref_rmsnorm", [REF / "kernels" / "rms-norm" / "rms_norm.cu"], COMMON)


# the reference's bench / test scripts that exercise the hot-path op surface (SURVEY Appendix B)
SCRIPT_FILES = [
    "kernels/hgemm/hgemm.py", "kernels/hgemm/tools/utils.py",
    "kernels/flash-attn/flash_attn_mma.py",
    "ffpa-attn/tests/test_ffpa_attn.py", "ffpa-attn/env.py",
    "kernels/sgemm/sgemm.py", "kernels/rope/rope.py", "kernels/rms-norm/rms_norm.py",
    "kernels/openai-triton/merge-attn-states/test_merge_attn_states.py",
    "kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.py",
    "kernels/openai-triton/merge-attn-states/triton_merge_attn_states.py",
]


def stage_scripts():
    """Copy the scripts (unmodified) to oracle/_ref/scripts/<same relative path>."""
    import shutil
    dst_root = OUT / "scripts"
    for rel in SCRIPT_FILES:
        src = REF / rel
        dst = dst_root / rel
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copyfile(src, dst)
    return dst_root


def load_prebuilt(name: str):
    """Import an already built oracle/_ref module (used on the GPU box, where
    no reference checkout is configured).  Returns None if it was never built."""
    import importlib.util
    so = OUT / name / f"{name}.so"
    if not so.exists():
        return None
    import torch  # noqa: F401  (the module links against libtorch)
    spec = importlib.util.spec_from_file_location(name, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    if not reference_present():
        print(f"no reference checkout at {REF} (set LEETCUDA_REFERENCE): nothing to build, a prebuilt oracle/_ref is used as is")
        sys.exit(0)
    which = sys.argv[1:] or ["hgemm", "fa", "ffpa", "sgemm", "merge", "rope", "rmsnorm", "scripts"]
    for w in which:
        {"hgemm": build_hgemm, "fa": build_fa, "ffpa": build_ffpa, "sgemm": build_sgemm,
         "merge": build_merge, "rope": build_rope, "rmsnorm": build_rmsnorm, "scripts": stage_scripts}[w]()
        print("built", w)
