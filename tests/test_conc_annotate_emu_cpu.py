"""CPU: tests/test_gpu_conc_annotate.py on the host emulation of the kernel sources (tests/host_emu, built by
conc_annotate.mk with the concordance handle): the annotation kernel and its C ABI against the reference's golden and the oracle, without a GPU.  The metrics test is left out: the
metrics pipeline is CUB and is not emulated."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "conc", "libugvc_emu_conc.so")


def test_annotation_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR, "-f", "conc_annotate.mk"], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "not metrics",
           "tests/test_gpu_conc_annotate.py"]
    run = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail
