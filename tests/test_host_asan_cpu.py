"""The host-side parsers that read untrusted bytes - filter-tree program compiler with its regexp compiler, the bytes-block / ZSTD
header walk and the part directory reader - built with AddressSanitizer + UndefinedBehaviorSanitizer (tests/host_asan/harness.cpp) and fed mutated real inputs.
Any out-of-bounds read, overflow, leak-on-throw or foreign exception type fails the run."""
import os
import shutil
import subprocess

import pytest

from victorialogs_b200 import scan as vs
from golden_util import load_filter_cases, build_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    out = tmp_path_factory.mktemp("asan") / "harness"
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
           "-I", os.path.join(ROOT, "victorialogs_b200", "csrc"), os.path.join(ROOT, "tests", "host_asan", "harness.cpp"), "-o", str(out), "-l:libzstd.so.1"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    if r.returncode != 0 and "sanitize" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    return str(out)


def run(harness, mode, seed_dir, iters, seed):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([harness, mode, str(seed_dir), str(iters), str(seed)], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, (r.returncode, r.stdout[-300:], r.stderr[-4000:])
    ok, bad = (int(x) for x in r.stdout.split()[1::2])
    return ok, bad


def test_program_compiler_under_sanitizers(harness, tmp_path):
    seeds = [build_filter(vs.Filter, c["filter"]).blob for c in load_filter_cases()[::5]]
    nxt = ("exact_prefix", "len_range", "string_range", "ipv4_range", "value_type")
    seeds += [build_filter(vs.Filter, c["filter"]).blob for c in load_filter_cases("filter_cases_next.json") if c["filter"]["kind"] in nxt][::4]
    seeds.append(vs.Filter.and_([vs.Filter.phrase("a", "b c"), vs.Filter.or_([vs.Filter.regexp("x", "a.*b|c+"), vs.Filter.not_(vs.Filter.in_("y", ["1", "2"]))])]).blob)
    seeds.append(vs.Filter.regexp("_msg", "(?i)^(foo|ba[rz]+)\\d{2,5}[^a-c]*.+$").blob)
    for i, s in enumerate(seeds):
        (tmp_path / ("%04d" % i)).write_bytes(s)
    ok, bad = run(harness, "tree", tmp_path, 60000, 1)
    assert ok > 1000 and bad > 10000


def test_zstd_header_walk_under_sanitizers(harness, tmp_path, oracle):
    k = 0
    for rpb in (3000, 64, 9000):       # one ZSTD block per frame / plain containers / several ZSTD blocks per frame
        cfg = oracle.GenConfig(seed=3, total_rows=rpb * 4, rows_per_block=rpb, hot_block_permille=500, hit_row_permille=60, columns_mask=0b1111)
        for b in range(4):
            for c in oracle.Block.generated(cfg, b).columns:
                (tmp_path / ("%04d" % k)).write_bytes(c.values_block)
                k += 1
    assert k >= 40
    ok, bad = run(harness, "zstd", tmp_path, 40000, 2)
    assert ok > 1000 and bad > 10000


def test_part_reader_under_sanitizers(harness, tmp_path):
    from test_part_reader_cpu import write_part
    path, files, originals, header = write_part(tmp_path, "part", seed=3)
    ok, bad = run(harness, "part", path, 4000, 3)
    assert ok > 200 and bad > 2000


def test_threaded_header_walk_under_thread_sanitizer(tmp_path, oracle):
    """tests/host_asan/walk_tsan.cpp: the multi-threaded walk (csrc/vl_zstd_job.h) over ~100 k values blocks on 1..33 threads under
    ThreadSanitizer: no data race, one digest, one first error."""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    exe = tmp_path / "walk_tsan"
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-fno-omit-frame-pointer", "-pthread", "-I", os.path.join(ROOT, "victorialogs_b200", "csrc"),
                        os.path.join(ROOT, "tests", "host_asan", "walk_tsan.cpp"), "-o", str(exe)], capture_output=True, text=True, timeout=300)
    if r.returncode != 0 and "tsan" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("ThreadSanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    seeds = tmp_path / "seeds"
    seeds.mkdir()
    k = 0
    for rpb in (3000, 64, 9000):
        cfg = oracle.GenConfig(seed=3, total_rows=rpb * 4, rows_per_block=rpb, hot_block_permille=500, hit_row_permille=60, columns_mask=0b1111)
        for b in range(4):
            for c in oracle.Block.generated(cfg, b).columns:
                (seeds / ("%04d" % k)).write_bytes(c.values_block)
                k += 1
    r = subprocess.run([str(exe), str(seeds), "2000"], capture_output=True, text=True, timeout=600, env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-4000:])
    assert "ok groups=" in r.stdout and int(r.stdout.rsplit("=", 1)[1]) >= 2      # the run crossed launch-group boundaries
    assert "WARNING: ThreadSanitizer" not in r.stderr


def test_host_pool_under_thread_sanitizer(tmp_path):
    """tests/host_asan/pool_tsan.cpp: the persistent packing threads of a ctx (csrc/vl_hostpool.h), thousands of jobs of 1..33 indices back to back."""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    exe = tmp_path / "pool_tsan"
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-fno-omit-frame-pointer", "-pthread", "-I", os.path.join(ROOT, "victorialogs_b200", "csrc"),
                        os.path.join(ROOT, "tests", "host_asan", "pool_tsan.cpp"), "-o", str(exe)], capture_output=True, text=True, timeout=300)
    if r.returncode != 0 and "tsan" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("ThreadSanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe), "3000"], capture_output=True, text=True, timeout=600, env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, (r.returncode, r.stdout[-500:], r.stderr[-4000:])
    assert r.stdout.startswith("ok total=") and "WARNING: ThreadSanitizer" not in r.stderr


def test_next_predicates_build_as_device_code(tmp_path):
    """csrc/vl_anycase.cuh is host+device: its host builds are checked against the oracle (tests/test_abi_cpu.py); here nvcc has to accept
    the same functions inside a kernel for sm_90a - no stack frame, no spills."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcudafe", "--diag_suppress=177", "-Xptxas", "-v",
                        "-I", os.path.join(ROOT, "victorialogs_b200", "csrc"), "-c", os.path.join(ROOT, "tests", "host_asan", "anycase_kernel.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in r.stderr


def test_value_predicates_under_sanitizers(harness, tmp_path):
    """the per-value predicates and number formatters of the row kernels (host builds of vl_hd.cuh / vl_anycase.cuh) on random values in
    exact-size heap blocks: what the device runs on every log value must not read a byte outside the value or the needle"""
    ok, bad = run(harness, "pred", tmp_path, 400000, 4)
    assert ok == 400000
