"""CPU: the calibrate_bridging_snvs kernels on the host emulation of their source (tests/host_emu, built by
bridging_snvs.mk): the test_hook_* tests of tests/test_gpu_bridging_snvs.py -- decide, scan and copy against the oracle
on the crafted corpus, every error reason and 100 k random records -- without a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "bsn", "libugvc_emu_bsn.so")


def test_kernels_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR, "-f", "bridging_snvs.mk"], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "hook",
           "tests/test_gpu_bridging_snvs.py"]
    run = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail
