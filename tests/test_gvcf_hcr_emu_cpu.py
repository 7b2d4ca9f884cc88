"""CPU: the gvcf_hcr kernels on the host emulation of their source (tests/host_emu, built by gvcf_hcr.mk): the
test_hook_* tests of tests/test_gpu_gvcf_hcr.py -- scan and emit against the oracle on the crafted corpus, every error
reason, about 200 k generated records, records without reset points shorter and longer than the segment bound, and
every cut of a record list into two pieces joined by the entry state -- without a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "hcr", "libugvc_emu_hcr.so")


def test_kernels_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR, "-f", "gvcf_hcr.mk"], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "hook",
           "tests/test_gpu_gvcf_hcr.py"]
    run = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail
