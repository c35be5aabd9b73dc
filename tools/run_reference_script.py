"""Run one of the reference's own bench / test scripts UNMODIFIED against the H100 kernels.

    python tools/run_reference_script.py <script.py> [script args...]
    python tools/run_reference_script.py --pytest <test_file.py> [pytest args...]

e.g.              python tools/run_reference_script.py $LEETCUDA_REFERENCE/kernels/hgemm/hgemm.py --MNK 8192 --mma --i 20
     (GPU box)    python tools/run_reference_script.py oracle/_ref/scripts/kernels/hgemm/hgemm.py --MNK 8192 --mma --i 20
                  (oracle/build_ref.py scripts stages the unmodified scripts there)

The scripts locate their extension by module name (SURVEY.md Appendix B): `toy_hgemm`, JIT
`flash_attn_lib`, `ffpa_attn` / `pyffpa_cuda`, JIT `sgemm_lib` (kernels/sgemm/sgemm.py:11), JIT
`merge_attn_states_cuda` (kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.py:6), JIT `rope`
(kernels/rope/rope.py:10), JIT `rms_norm_lib` (kernels/rms-norm/rms_norm.py:10).  This
launcher registers the mirrors under those names and intercepts torch.utils.cpp_extension.load for
them, changes into the script's directory (the scripts use relative imports such as `../env.py`),
then runs the script as __main__ (or hands the file to pytest in this process).
"""
import os
import runpy
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch.utils.cpp_extension as ext  # noqa: E402

import leetcuda_b200.ffpa_attn  # noqa: E402
import leetcuda_b200.flash_attn  # noqa: E402
import leetcuda_b200.hgemm  # noqa: E402
import leetcuda_b200.merge_attn_states  # noqa: E402
import leetcuda_b200.rms_norm  # noqa: E402
import leetcuda_b200.rope  # noqa: E402
import leetcuda_b200.sgemm  # noqa: E402

MIRRORS = {
    "toy_hgemm": leetcuda_b200.hgemm, "hgemm_lib": leetcuda_b200.hgemm,
    "flash_attn_lib": leetcuda_b200.flash_attn,
    "ffpa_attn": leetcuda_b200.ffpa_attn, "pyffpa_cuda": leetcuda_b200.ffpa_attn,
    "sgemm_lib": leetcuda_b200.sgemm,
    "merge_attn_states_cuda": leetcuda_b200.merge_attn_states.lib,
    "rope": leetcuda_b200.rope, "rms_norm_lib": leetcuda_b200.rms_norm,
}
for _name in ("toy_hgemm", "ffpa_attn", "pyffpa_cuda"):
    sys.modules[_name] = MIRRORS[_name]

_orig_load = ext.load


def _load(name, *args, **kwargs):
    if name in MIRRORS:
        print(f"[leetcuda_b200] serving extension '{name}' from the sm_90a mirror", flush=True)
        return MIRRORS[name]
    return _orig_load(name, *args, **kwargs)


ext.load = _load

if __name__ == "__main__":
    argv = sys.argv[1:]
    use_pytest = bool(argv) and argv[0] == "--pytest"
    if use_pytest:
        argv = argv[1:]
    if not argv:
        sys.exit(__doc__)
    script = os.path.abspath(argv[0])
    os.chdir(os.path.dirname(script))
    sys.path.insert(0, os.path.dirname(script))
    if use_pytest:
        import pytest
        sys.exit(pytest.main([script, "-p", "no:cacheprovider", *argv[1:]]))
    sys.argv = [script, *argv[1:]]
    runpy.run_path(script, run_name="__main__")
