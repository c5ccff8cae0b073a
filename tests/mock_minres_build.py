"""TEST INFRASTRUCTURE ONLY: tests/mock_build.py's host-memory mock with the fused MINRES entry
points restated (tests/mock/mock_fused_minres.c, which compiles mock_base.c into itself), linked
with the C++ host layer into one DSO.  Used by tests/test_fused_minres_cpu.py and, with
B200_TEST_SELFCHECK=1, by tests/test_fused_minres_gpu.py."""
import ctypes
import os
import subprocess

from tests.mock_build import ROOT, link_args

MOCK_DIR = os.path.join(ROOT, "tests", "mock")
NAMES = ["b200_minres_fused_%s_%s" % (n, v) for n in ("work_size", "init", "lanczos", "update")
         for v in ("f64", "f32")] + \
        ["b200_csr_spmv_sub_dot_%s_%s" % (v, i) for v in ("f64", "f32") for i in ("i32", "i64")]


def build_mock_host(d):
    from ginkgo_b200 import api
    inc = os.path.join(ROOT, "include")
    # gen_mock.py writes a stub for every declared entry point it does not find defined in the file it
    # is given: mock_base.c plus the names mock_fused_minres.c defines through its macros
    listed = os.path.join(d, "handwritten.c")
    with open(os.path.join(MOCK_DIR, "mock_base.c")) as f, open(listed, "w") as out:
        out.write(f.read() + "".join("\n%s();" % n for n in NAMES))
    gen = os.path.join(d, "mock_gen.c")
    subprocess.run(["python", os.path.join(MOCK_DIR, "gen_mock.py"), os.path.join(inc, "ginkgo_b200.h"),
                    os.path.join(ROOT, "oracle", "liboracle.so"), listed, gen], check=True, capture_output=True)
    objs = []
    for src in (os.path.join(MOCK_DIR, "mock_fused_minres.c"), gen):
        o = os.path.join(d, os.path.basename(src) + ".o")
        subprocess.run(["gcc", "-O1", "-fPIC", "-I" + inc, "-c", src, "-o", o], check=True)
        objs.append(o)
    so = os.path.join(d, "libgko_b200_host_mock_minres.so")
    # one DSO, -Bsymbolic: the b200_* references of the host layer bind to the mock inside it
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-o", so,
                    os.path.join(ROOT, "ginkgo_b200", "host", "capi.cpp")] + objs + link_args(), check=True)
    return api._configure_host_lib(ctypes.CDLL(so))
