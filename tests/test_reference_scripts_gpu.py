"""The reference's own bench / test scripts, UNMODIFIED, against the sm_90a mirror (north_star: "drop-in
replacements callable from the existing bench scripts"; SURVEY Appendix B).

`python oracle/build_ref.py scripts` stages the scripts byte for byte under oracle/_ref/scripts/ (git-ignored,
the tests skip where they have not been staged).
tools/run_reference_script.py injects the mirror modules under the names the scripts load
(toy_hgemm, flash_attn_lib, ffpa_attn, sgemm_lib, merge_attn_states_cuda) and runs them.  The tests assert
on the scripts' own output: their `all close: True` lines (flash_attn_mma.py:465-494,
test_ffpa_attn.py:583-614), the TFLOPS rows of hgemm.py:281-329, and the reference's pytest for
merge_attn_states (test_merge_attn_states.py:95-300).  The printed tables are written to
ref_scripts_*.log in the system temp directory.
"""
import os
import re
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
SCRIPTS = ROOT / "oracle" / "_ref" / "scripts"
LAUNCH = ROOT / "tools" / "run_reference_script.py"


def _run(rel, *args, pytest_mode=False, timeout=900, log=None):
    script = SCRIPTS / rel
    if not script.exists():
        pytest.skip(f"{script} not staged (python oracle/build_ref.py scripts)")
    cmd = [sys.executable, str(LAUNCH)] + (["--pytest"] if pytest_mode else []) + [str(script), *args]
    env = dict(os.environ, PYTHONUNBUFFERED="1", TORCH_CUDA_ARCH_LIST="9.0a")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)
    text = r.stdout + "\n" + r.stderr[-4000:]
    if log:
        out = Path(tempfile.gettempdir())
        (out / log).write_text("$ " + " ".join(cmd[1:]) + "\n" + r.stdout + ("\n[stderr tail]\n" + r.stderr[-2000:] if r.returncode else ""))
    assert r.returncode == 0, text[-3000:]
    return r.stdout


def test_hgemm_script_small_and_headline():
    """kernels/hgemm/hgemm.py — BASELINE configs[0] (512^3) and configs[1] (8192^3), every tensor-core family."""
    out = _run("kernels/hgemm/hgemm.py", "--MNK", "512", "--mma", "--mma-tn", "--cute-tn", "--wmma", "--show-all-info", "--i", "5",
               log="ref_scripts_hgemm_512.log")
    assert len(re.findall(r"TFLOPS:\s*[0-9.]+", out)) >= 3, out[-2000:]
    out = _run("kernels/hgemm/hgemm.py", "--MNK", "8192", "--mma", "--mma-tn", "--cute-tn", "--wmma", "--show-all-info", "--i", "20",
               log="ref_scripts_hgemm_8192.log")
    tf = [float(x) for x in re.findall(r"TFLOPS:\s*([0-9.]+)", out)]
    assert tf and max(tf) > 300.0, out[-2000:]         # the script's own host-clock TFLOPS of the wgmma kernel


def test_flash_attn_script_check():
    """kernels/flash-attn/flash_attn_mma.py --check at BASELINE configs[2]: every `all close` line must be True."""
    out = _run("kernels/flash-attn/flash_attn_mma.py", "--B", "4", "--H", "32", "--N", "4096", "--D", "128",
               "--check", "--show-all", "--iters", "20", "--seed", "1", log="ref_scripts_flash_attn_B4H32N4096D128.log")
    assert "serving extension 'flash_attn_lib'" in out
    checks = re.findall(r"all close:\s*(\w+)", out)
    assert len(checks) >= 6, out[-3000:]
    assert all(c == "True" for c in checks), [ln for ln in out.splitlines() if "all close" in ln]
    tf = [float(x) for x in re.findall(r"TFLOPS:\s*([0-9.]+)", out)]
    assert tf and max(tf) > 800.0, out[-2000:]


def test_ffpa_script_check():
    """ffpa-attn/tests/test_ffpa_attn.py --check at BASELINE configs[3] (B2 H16 N2048 D512)."""
    out = _run("ffpa-attn/tests/test_ffpa_attn.py", "--B", "2", "--H", "16", "--N", "2048", "--D", "512",
               "--check", "--show-all", "--iters", "20", log="ref_scripts_ffpa_B2H16N2048D512.log")
    checks = re.findall(r"all close:\s*(\w+)", out)
    assert len(checks) >= 2, out[-3000:]
    assert all(c == "True" for c in checks), [ln for ln in out.splitlines() if "all close" in ln]


def test_merge_attn_states_reference_pytest():
    """The only pytest of the reference that covers an op of this path, run as is against the mirror
    (kernels/openai-triton/merge-attn-states/test_merge_attn_states.py): 15 parametrised cases."""
    out = _run("kernels/openai-triton/merge-attn-states/test_merge_attn_states.py", "-q", "-x", pytest_mode=True,
               log="ref_scripts_merge_pytest.log")
    m = re.search(r"(\d+) passed", out)
    assert m and int(m.group(1)) >= 15, out[-3000:]
    assert "failed" not in out.split("passed")[-1]


def _first_values(out):
    """`out_<tag>: ['v0', 'v1', 'v2'], time:...` lines of rope.py / rms_norm.py -> [(tag, [v0, v1, v2])] in print order."""
    rows = []
    for m in re.finditer(r"out_(\w+): \[([^\]]*)\], time", out):
        vals = [float(x.strip().strip("'")) for x in m.group(2).split(",")]
        rows.append((m.group(1), vals))
    return rows


def test_rope_script():
    """kernels/rope/rope.py as is: per shape it prints the first three outputs of rope_f32, rope_f32x4_pack and its own
    torch implementation (naive_rope) — they must agree."""
    out = _run("kernels/rope/rope.py", log="ref_scripts_rope.log")
    assert "serving extension 'rope'" in out
    rows = _first_values(out)
    assert len(rows) == 12, out[-2000:]          # 4 shapes x (f32, f32x4_pack, f32_th)
    for i in range(0, len(rows), 3):
        (_, a), (_, b), (tag, th) = rows[i:i + 3]
        assert tag == "f32_th"
        for x, y, z in zip(a, b, th):
            assert abs(x - z) < 1e-4 and abs(y - z) < 1e-4, rows[i:i + 3]


def test_rms_norm_script():
    """kernels/rms-norm/rms_norm.py as is: every op's first three outputs against the script's torch row of the same
    block (the script's "f16 overflow without f32" blocks scale x by 100 to show its fp16-statistics kernels
    overflowing; the ops here keep fp32 statistics under every name, so they must match the fp32 row there too)."""
    out = _run("kernels/rms-norm/rms_norm.py", log="ref_scripts_rms_norm.log")
    assert "serving extension 'rms_norm_lib'" in out
    rows = _first_values(out)
    assert len(rows) >= 20, out[-2000:]
    block = []
    checked = 0
    for tag, vals in rows:
        if tag.endswith("_th"):
            if all(abs(v) > 0 and v == v for v in vals):      # torch fp16 row of the overflow block is nan / 0: skip it
                for t, got in block:
                    tol = 1e-5 if t.startswith("f32") else 2e-3
                    assert all(abs(g - w) <= tol * max(1.0, abs(w)) for g, w in zip(got, vals)), (t, got, vals)
                    checked += 1
            block = []
        else:
            block.append((tag, vals))
    assert checked >= 12
