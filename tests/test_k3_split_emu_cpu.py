"""CPU: tests/test_gpu_k3_split.py on the host emulation of the kernel sources (tests/host_emu), where one thread plays
both threads of a record, B then A, through k3_heap_split's hand-over code: the split form against the one-thread
k3_heap, bit for bit, without a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "libugvc_emu.so")


def test_split_hand_over_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_k3_split.py"]
    run = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail
