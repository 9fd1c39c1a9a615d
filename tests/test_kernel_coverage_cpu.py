"""Every kernel template instantiation in the built library is run by a GPU test (no GPU needed here).

A launcher picks among instantiations by shape, and an instantiation that no test runs can be wrong while the suite
stays green.  This lists the library's kernel entry points (cuobjdump -symbols, demangled by cu++filt) and requires
each template instantiation to be a key of test_gpu_shape_edges.COVERS -- whose GPU cases assert under torch.profiler
that they launched it -- or to be listed, with a reason, in its EXEMPT (by instantiation or by kernel name).  A kernel
that is not a template has one instantiation, which every call of its entry point runs."""
import os
import shutil
import subprocess

import pytest

import test_gpu_shape_edges as E


def _cuda_tool(name):
    for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if root and os.path.exists(os.path.join(root, "bin", name)):
            return os.path.join(root, "bin", name)
    return shutil.which(name)


def _instantiations():
    dump, filt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    if dump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: cannot list the library's kernels")
    from mgproto_b200.build import build
    lib = build()
    sym = subprocess.run([dump, "-symbols", lib], capture_output=True, text=True, check=True).stdout
    mangled = sorted({ln.split()[-1] for ln in sym.splitlines() if "STO_ENTRY" in ln})
    assert mangled, "no kernel entry points found in %s" % lib
    names = subprocess.run([filt], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
    return {E.kernel_key(n) for n in names.splitlines() if n.strip()}


def test_kernel_key_normalises_both_demanglers():
    assert E.kernel_key("void <unnamed>::head_top1_kernel<(int)32, (int)1, (int)256>(const unsigned long long *, int)") \
        == "head_top1_kernel<32, 1, 256>"
    assert E.kernel_key("void (anonymous namespace)::em_tc_kernel<128, 16>(CUtensorMap_st, "
                        "(anonymous namespace)::EmTcParams)") == "em_tc_kernel<128, 16>"
    assert E.kernel_key("void <unnamed>::normalize_fwd_kernel<__nv_bfloat16, (bool)1>(const T1 *, float *)") \
        == "normalize_fwd_kernel<__nv_bfloat16, true>"
    assert E.kernel_key("<unnamed>::proto_weight_kernel(const float *, int)") == "proto_weight_kernel"


def test_every_kernel_instantiation_is_covered():
    kernels = _instantiations()
    inst = sorted(k for k in kernels if "<" in k)
    assert inst, "no template instantiations found"
    missing = [k for k in inst if k not in E.COVERS and k not in E.EXEMPT and k.split("<")[0] not in E.EXEMPT]
    assert not missing, ("kernel instantiations that no GPU test runs (add a case to tests/test_gpu_shape_edges.py "
                         "and a COVERS entry, or an EXEMPT entry with the reason): %s" % missing)
    stale = sorted(set(E.COVERS) - kernels)
    assert not stale, "COVERS names instantiations the library does not have: %s" % stale
