"""The C-ABI library loads without a GPU and exports every symbol include/leetcuda_b200.h declares."""
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def declared_symbols():
    text = (ROOT / "include" / "leetcuda_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_expected_entry_points():
    syms = declared_symbols()
    for s in ["b200_version", "b200_last_error", "b200_launch_count", "b200_hgemm_f16",
              "b200_hgemm_f16_ex", "b200_hgemm_f16_acc16", "b200_hgemm_f16_rows", "b200_hgemm_f16_rows_fused", "b200_fmha_fwd_f16",
              "b200_hgemm_f16_host", "b200_fmha_fwd_f16_host", "b200_sgemm_tf32", "b200_sgemm_tf32_ex",
              "b200_tf32_round_inplace", "b200_merge_attn_states"]:
        assert s in syms


def test_library_exports_every_declared_symbol(built_lib):
    for s in declared_symbols():
        assert hasattr(built_lib, s), f"{s} declared in the header but not exported"


def test_ctypes_signatures_cover_header(built_lib):
    from leetcuda_b200 import _capi
    assert sorted(_capi.SIGNATURES) == declared_symbols()


def test_version_and_error_text(built_lib):
    assert built_lib.b200_version() == 1000
    assert isinstance(built_lib.b200_last_error(), bytes)


def test_argument_validation_without_gpu(built_lib):
    """Bad arguments are rejected before any CUDA call is made."""
    from leetcuda_b200 import _capi
    rc = built_lib.b200_hgemm_f16(None, None, None, 128, 128, 128, 0, None)
    assert rc == -1 and "null" in _capi.last_error()
    rc = built_lib.b200_hgemm_f16(16, 16, 16, 128, 100, 128, 0, None)  # N % 8 != 0
    assert rc == -1 and "multiples of 8" in _capi.last_error()
    rc = built_lib.b200_hgemm_f16(16, 16, 16, 128, 128, 128, 7, None)
    assert rc == -1 and "b_layout" in _capi.last_error()
    rc = built_lib.b200_sgemm_tf32(16, 16, 16, 128, 128, 126, 0, 0, None)   # K % 4 != 0
    assert rc == -1 and "multiples of 4" in _capi.last_error()
    rc = built_lib.b200_sgemm_tf32(None, 16, 16, 128, 128, 128, 0, 1, None)
    assert rc == -1
    rc = built_lib.b200_tf32_round_inplace(8, 16, None)                      # misaligned pointer
    assert rc == -1 and "aligned" in _capi.last_error()
    rc = built_lib.b200_merge_attn_states(16, None, 16, 16, 16, 16, 4, 2, 12, 1, None)   # 12 % 8 != 0
    assert rc == -1 and "headsize must be multiple of pack_size:8" in _capi.last_error()
    rc = built_lib.b200_merge_attn_states(16, None, 16, 16, 16, 16, 4, 2, 16, 9, None)
    assert rc == -3 and "Unsupported data type of O" in _capi.last_error()
    rc = built_lib.b200_fmha_fwd_f16(16, 16, 16, 16, 1, 1, 128, 100, 0, 0.0, None)
    assert rc == -3 and "headdim not support" in _capi.last_error()
    rc = built_lib.b200_fmha_fwd_f16(16, 16, 16, 16, 0, 1, 128, 128, 0, 0.0, None)
    assert rc == -1


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from leetcuda_b200 import _capi
    monkeypatch.setattr(_capi, "_lib", None)
    monkeypatch.setenv("LEETCUDA_B200_LIB", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no fallback"):
        _capi.lib()


def test_sass_is_hopper_native(built_lib):
    """wgmma / TMA / mbarrier opcodes are present in the shipped SASS (HGMMA, UTMALDG, SYNCS)."""
    import shutil
    import subprocess
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", str(_capi.LIB_PATH)], capture_output=True, text=True).stdout
    for op in ("HGMMA", "UTMALDG", "SYNCS"):
        assert op in sass, op
    assert "HMMA.16816" not in sass  # no legacy mma.sync path
