"""Link-level drop-in proof: a C++ translation unit that includes the reference's OWN headers
(cudamat/cudamat_conv_gemm.cuh, cudamat/cudamat_conv.cuh) links against the product under the library names the
reference's Makefile uses (`-lcudamat_conv_gemm -lcudamat_conv`, Makefile:72-77), and — on the GPU box — computes
the right numbers through both symbol sets.  The binary is built where /root/reference exists (here) and travels."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "drop_in", "link_drop_in.cc")
BIN = os.path.join(ROOT, "tests", "drop_in", "_build", "link_drop_in")
REF = "/root/reference/cudamat"


def build_drop_in():
    """g++ with the reference's header directory; rpath points at convnet_b200/lib relative to the binary.
    Two binaries: one linked with -lcudamat_conv_gemm only, one with -lcudamat_conv only (both names are aliases of
    the one product library, so either must resolve BOTH symbol sets the program calls)."""
    from convnet_b200 import build
    lib = build.build()
    libdir = os.path.dirname(lib)
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    outs = []
    for alias in ("cudamat_conv_gemm", "cudamat_conv"):
        out = BIN + "_" + alias
        cmd = ["g++", "-O1", "-std=c++14", "-I" + REF, "-I/usr/local/cuda/include", SRC, "-o", out,
               "-L" + libdir, "-l" + alias, "-L/usr/local/cuda/lib64", "-lcudart",
               "-Wl,--no-undefined", "-Wl,-rpath,$ORIGIN/../../../convnet_b200/lib", "-Wl,-rpath,/usr/local/cuda/lib64"]
        subprocess.run(cmd, check=True)
        outs.append(out)
    return outs


@pytest.mark.skipif(not os.path.isdir(REF), reason="needs the reference headers under /root/reference")
def test_reference_headers_compile_and_link_against_the_product():
    for b, name in zip(build_drop_in(), ("libcudamat_conv_gemm.so", "libcudamat_conv.so")):
        out = subprocess.run(["ldd", b], capture_output=True, text=True).stdout
        line = [l for l in out.splitlines() if name in l]
        assert line and os.path.join("convnet_b200", "lib") in line[0], out
        # every reference prototype the program calls resolved to the product (-Wl,--no-undefined made the link fail otherwise)
        syms = subprocess.run(["nm", "-D", "--undefined-only", b], capture_output=True, text=True).stdout
        for s in ("convUpGemm", "convUp", "MaxPoolGemm", "MaxPool", "SetupTexture"):
            assert (" U %s\n" % s) in syms or (" U %s@" % s) in syms, (s, syms)


@pytest.mark.gpu
def test_drop_in_binary_runs_on_the_gpu():
    for alias in ("cudamat_conv_gemm", "cudamat_conv"):
        b = BIN + "_" + alias
        if not os.path.exists(b):
            pytest.skip("%s is built only where the reference's headers exist (__graft_entry__.build())" % b)
        r = subprocess.run([b], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "DROP-IN OK" in r.stdout, (r.returncode, r.stdout, r.stderr)
