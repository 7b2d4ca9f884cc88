"""CPU: the parity tests of the CUDA path, run on the kernel SOURCES compiled for the host.

tests/host_emu builds variantcalling_b200/csrc/kernels.cu (K1 field parse, K2 feature assembly, K3
inference) and capi.cu with g++ over a stand-in cuda_runtime.h -- one emulated thread per CTA, device
memory on the heap -- into tests/host_emu/_build/libugvc_emu.so.  This test points a child pytest at
that library (UGVC_LIB_PATH, the developer override of variantcalling_b200/lib.py) and runs the
`gpu`-marked parity files there, so the driver's CPU check already compares the code the GPU will
execute with the oracle: features bit-identical, FILTER identical, CLI output line for line, the
inputs the reference raises on, --treat_multiallelics (its kernels, csrc/multiallelic.cu, included), the fuzzed records.

Test infrastructure only: the package never loads the emulated library, and
tests/test_capi_cpu.py::test_no_cuda_device_fails_loudly keeps asserting that the product library
refuses to run without a CUDA device.  Not emulated (their tests stay GPU-only): K0's cooperative
tile scan (lines are indexed by a host loop with the same outputs and error codes), the device
synthetic generator and the concordance kernels (CUB pipelines)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "host_emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "libugvc_emu.so")

FILES = ["tests/test_gpu_parity.py", "tests/test_gpu_edges.py", "tests/test_gpu_fuzz.py", "tests/test_gpu_cnv.py",
         "tests/test_gpu_cli.py", "tests/test_gpu_multiallelics.py", "tests/test_gpu_x_model_apply.py", "tests/test_gpu_x_deepvariant.py", "tests/test_gpu_x_bgzf.py",
         "tests/test_gpu_x_inflate_edges.py", "tests/test_gpu_y_tiletok.py", "tests/test_gpu_feature_edges.py",
         "tests/test_gpu_y_deviations.py", "tests/test_gpu_z_multiallelic_device.py", "tests/test_gpu_k3_shapes.py"]
DEVICE_ONLY = ["tests/test_gpu_edges.py::test_device_generator_text_parity",  # the device synthetic generator
               "tests/test_gpu_parity.py::test_full_size_properties_batching_invariance",
               # the emulation compiles one k3_heap instantiation: forcing the others is a device matter
               "tests/test_gpu_k3_shapes.py::test_every_compiled_shape_scores_identically"]


def test_kernel_sources_pass_the_parity_suite_on_the_host_emulation():
    build = subprocess.run(["make", "-C", EMU_DIR], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB)
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", *FILES]
    for t in DEVICE_ONLY:
        cmd += ["--deselect", t]
    run = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0, tail
    assert " passed" in run.stdout and "failed" not in run.stdout.splitlines()[-1], tail


def test_two_rank_cli_run_equals_the_single_process_output(tmp_path):
    """`torchrun --nproc-per-node 2 ugvc filter_variants_pipeline ...`: ranks own whole contigs (LPT on the
    input's compressed spans), write BGZF parts, all-reduce the counters once (gloo here, NCCL on GPUs)
    and rank 0 splices the parts into one file + .tbi.  On the host emulation: same records, same
    order, a working index, global counts in the log."""
    import gzip
    import pickle

    from tests import util
    from variantcalling_b200 import bgzf_io

    build = subprocess.run(["make", "-C", EMU_DIR], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stderr[-3000:]
    ds = util.make_dataset(n_records=9000, n_custom=3, seed=77,
                           contigs={"chr1": 5_000_000, "chr2": 2_500_000, "chr3": 2_000_000, "chr4": 1_500_000, "chr5": 800_000})
    _, tr, x = util.fit_transformer(ds)
    model = util.fit_model("lr", x, ds["labels"])
    vcf, mpath = str(tmp_path / "in.vcf.gz"), str(tmp_path / "m.pkl")
    bgzf_io.write_vcf_gz(vcf, ds["header"], ds["lines"])
    with open(mpath, "wb") as fh:
        pickle.dump({"xgb": model, "transformer": tr}, fh)
    tool = ["filter_variants_pipeline", "--input_file", vcf, "--model_file", mpath, "--blacklist_cg_insertions",
            "--device", "0"]  # the emulation exposes one device (on a GPU box every rank takes LOCAL_RANK)
    for c in ds["customs"]:
        tool += ["--custom_annotations", c]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB, CUDA_VISIBLE_DEVICES="")  # gloo: both ranks share emulated device 0
    env.pop("RANK", None), env.pop("WORLD_SIZE", None)
    one, two = str(tmp_path / "one.vcf.gz"), str(tmp_path / "two.vcf.gz")
    r1 = subprocess.run([sys.executable, "ugvc", *tool, "--output_file", one], cwd=ROOT, env=env, capture_output=True,
                        text=True, timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    r2 = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                         "--master-addr", "127.0.0.1", "--master-port", "29731", "ugvc/__main__.py", *tool,
                         "--output_file", two], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r2.returncode == 0, r2.stderr[-4000:]
    assert gzip.open(two).read() == gzip.open(one).read()
    i1, i2 = bgzf_io.read_tbi(one + ".tbi"), bgzf_io.read_tbi(two + ".tbi")
    assert list(i1) == list(i2) == ["chr1", "chr2", "chr3", "chr4", "chr5"]
    for c in i1:
        assert bgzf_io.inflate(two, *i2[c]).tobytes() == bgzf_io.inflate(one, *i1[c]).tobytes()
    assert not [f for f in os.listdir(tmp_path) if ".part" in f]           # parts are cleaned up
    summary = [ln for ln in r1.stderr.splitlines() if "records written" in ln][0].split(" ", 2)[2]
    assert sum(summary in ln for ln in r2.stderr.splitlines()) == 2        # both ranks report the global counts
    assert "rank 0/2" in r2.stderr and "rank 1/2" in r2.stderr


def test_two_rank_run_of_the_multiallelic_branch(tmp_path):
    """--treat_multiallelics --recalibrate_genotype under two ranks: every rank builds its own device split plan for its
    contigs (csrc/multiallelic.cu on the emulation); the assembled file equals the single-process output byte for byte."""
    import gzip
    import pickle

    from tests import multiallelic_data as MD
    from tests import util
    from variantcalling_b200 import bgzf_io

    build = subprocess.run(["make", "-C", EMU_DIR], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stderr[-3000:]
    ds, tr, model, _split = util.make_multiallelic_case(21, "gb3")
    vcf, fasta, mpath = str(tmp_path / "in.vcf.gz"), str(tmp_path / "ref.fa"), str(tmp_path / "m.pkl")
    bgzf_io.write_vcf_gz(vcf, ds["header"], ds["lines"])
    with open(fasta, "w") as fh:
        fh.write(MD.fasta_text(ds["ref"]))
    with open(mpath, "wb") as fh:
        pickle.dump({"xgb": model, "transformer": tr}, fh)
    tool = ["filter_variants_pipeline", "--input_file", vcf, "--model_file", mpath, "--treat_multiallelics", "--ref_fasta", fasta,
            "--recalibrate_genotype", "--device", "0"]
    for c in ds["customs"]:
        tool += ["--custom_annotations", c]
    env = dict(os.environ, UGVC_LIB_PATH=EMU_LIB, CUDA_VISIBLE_DEVICES="")  # gloo: both ranks share emulated device 0
    env.pop("RANK", None), env.pop("WORLD_SIZE", None)
    one, two = str(tmp_path / "one.vcf.gz"), str(tmp_path / "two.vcf.gz")
    r1 = subprocess.run([sys.executable, "ugvc", *tool, "--output_file", one], cwd=ROOT, env=env, capture_output=True,
                        text=True, timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    r2 = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                         "--master-addr", "127.0.0.1", "--master-port", "29741", "ugvc/__main__.py", *tool,
                         "--output_file", two], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r2.returncode == 0, r2.stderr[-4000:]
    assert gzip.open(two).read() == gzip.open(one).read()
    assert "Processing multiallelics" in r2.stderr
