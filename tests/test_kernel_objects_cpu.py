"""The functions inside libvlscan.so, read with cuobjdump (no GPU needed): each is compiled into exactly one of the library's embedded cubins,
and every `__global__` defined under victorialogs_b200/csrc is among them.  nvcc emits a static kernel in every translation unit that
includes its definition, launched there or not, so a kernel header included by two .cu files doubles its kernels' build time and their
share of the library; this test fails on such an include."""
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "victorialogs_b200", "csrc")
LIB = os.path.join(ROOT, "victorialogs_b200", "libvlscan.so")


def cuda_tool(name):
    exe = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    return exe if os.path.exists(exe) else None


@pytest.fixture(scope="module")
def cubins():
    exe = cuda_tool("cuobjdump")
    if not os.path.exists(LIB) or exe is None:
        pytest.skip("needs victorialogs_b200/libvlscan.so and cuobjdump")
    r = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = []   # one list of function names per embedded cubin
    for line in r.stdout.splitlines():
        if line.startswith("Fatbin elf code"):
            out.append([])
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            assert out, "a function listed before any cubin"
            out[-1].append(m.group(1))
    assert len(out) >= 2
    return out


def source_kernels():
    """The names of the `__global__` functions defined under csrc."""
    names = set()
    for path in glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")):
        with open(path) as f:
            for line in f:
                if "__global__" in line and not line.lstrip().startswith("//"):
                    m = re.search(r"\b(k_\w+)\s*\(", line)
                    assert m, (path, line)
                    names.add(m.group(1))
    assert len(names) > 40
    return names


def kernel_names(mangled):
    """The function name of each mangled name (cu++filt), e.g. `k_hits_group` for `void vl::k_hits_group<(bool)0>(...)`, or None when it is
    not a `k_...` function."""
    exe = cuda_tool("cu++filt")
    if exe is None:
        pytest.skip("needs cu++filt")
    r = subprocess.run([exe], input="\n".join(mangled) + "\n", capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    out = r.stdout.splitlines()
    assert len(out) == len(mangled)
    names = []
    for d in out:
        m = re.search(r"(?:^|[\s:>])(k_\w+)(?=[<(])", d)
        names.append(m.group(1) if m else None)
    return names


def test_kernel_names_are_exact():
    # a kernel whose name is a prefix of another's must not be taken for it, nor the other way round
    assert kernel_names(["_ZN2vl18k_facets_formattedENS_9BatchViewEPKjjiPj", "_ZN2vl8k_facetsENS_9BatchViewENS_10FacetsArgsEPy",
                         "_ZN2vl12k_hits_groupILb0EEEvNS_9BatchViewENS_9HitsQueryENS_8HitsViewENS_9HitsTableEPKjPKmPy",
                         "_ZN41_GLOBAL__N__d99cc33f_9_vl_gen_cu_23d1f10110k_gen_pokeEPhPKmPKhm"]) == \
        ["k_facets_formatted", "k_facets", "k_hits_group", "k_gen_poke"]


def test_every_function_is_in_one_cubin(cubins):
    where = {}
    for i, funcs in enumerate(cubins):
        for fn in set(funcs):
            where.setdefault(fn, []).append(i)
    dup = sorted(fn for fn, at in where.items() if len(at) > 1)
    assert not dup, "%d functions compiled into more than one translation unit: %s" % (len(dup), ", ".join(dup))


def test_every_source_kernel_is_compiled(cubins):
    found = set(kernel_names([fn for funcs in cubins for fn in funcs]))
    missing = sorted(source_kernels() - found)
    assert not missing, "kernels defined under csrc but absent from libvlscan.so: %s" % ", ".join(missing)
