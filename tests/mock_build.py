"""TEST INFRASTRUCTURE ONLY: builds the C++ host layer (ginkgo_b200/host/capi.cpp) together with
tests/mock -- the host-memory stand-in for the C ABI whose kernel entry points forward to the
oracle, with the fused solver kernels restated by hand -- into one DSO and wraps it for
ginkgo_b200.api.  Used by tests/test_host_cpu.py, the tests/test_fused_*_cpu.py files and, with
B200_TEST_SELFCHECK=1, as a stand-in for the GPU executor when the bodies of the gpu tests are
checked on a machine without a GPU."""
import ctypes
import glob
import os
import subprocess

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK_DIR = os.path.join(ROOT, "tests", "mock")


class CpuExec:
    """stands where api.HostExecutor stands: a gkob executor handle on the mock"""

    def __init__(self, lib):
        self.h = lib.gkob_exec_create(0, None)
        assert self.h
        self.device = torch.device("cpu")
        self.stream = None
        self._lib = lib

    def synchronize(self):
        pass

    def launch_count(self):
        return self._lib.gkob_launch_count(self.h)


def build_mock_objects(d, sanitize=()):
    """the handwritten tests/mock/*.c + the generated forwarders, compiled into `d`; returns the object
    files"""
    inc = os.path.join(ROOT, "include")

    def compile_c(src):
        o = os.path.join(d, os.path.basename(src) + ".o")
        subprocess.run(["gcc", "-O1", "-fPIC", "-I" + inc, "-c", src, "-o", o] + list(sanitize), check=True)
        return o

    objs = [compile_c(src) for src in sorted(glob.glob(os.path.join(MOCK_DIR, "*.c")))]
    # gen_mock.py forwards or stubs every entry point these objects do not define
    handwritten = set()
    for o in objs:
        for line in subprocess.run(["nm", "-g", "--defined-only", o], check=True, capture_output=True,
                                   text=True).stdout.splitlines():
            parts = line.split()
            if len(parts) == 3 and parts[2].startswith("b200_"):
                handwritten.add(parts[2])
    gen = os.path.join(d, "mock_gen.c")
    subprocess.run(["python", os.path.join(MOCK_DIR, "gen_mock.py"), os.path.join(inc, "ginkgo_b200.h"),
                    os.path.join(ROOT, "oracle", "liboracle.so"), gen] + sorted(handwritten), check=True,
                   capture_output=True)
    return objs + [compile_c(gen)]


def link_args():
    return ["-L" + os.path.join(ROOT, "oracle"), "-loracle", "-lpthread", "-lm",
            "-Wl,-rpath," + os.path.join(ROOT, "oracle")]


def build_mock_executable(d, source, name):
    """a C++ program written against the host layer, linked with the mock instead of the CUDA library"""
    exe = os.path.join(d, name)
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", source] + build_mock_objects(d) + link_args() +
                   ["-o", exe], check=True)
    return exe


def build_mock_host(d):
    from ginkgo_b200 import api
    # B200_MOCK_SANITIZE=1: build the host layer + mock with ASan / UBSan; run pytest with
    # LD_PRELOAD="$(g++ -print-file-name=libasan.so) $(g++ -print-file-name=libstdc++.so)" and
    # ASAN_OPTIONS=detect_leaks=0 (the preload also reaches gcc and python, whose exit-time leaks
    # would fail the build)
    san = (["-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-g"]
           if os.environ.get("B200_MOCK_SANITIZE") == "1" else [])
    objs = build_mock_objects(d, san)
    so = os.path.join(d, "libgko_b200_host_mock.so")
    # one DSO, -Bsymbolic: the b200_* references of the host layer bind to the mock inside it,
    # whatever else the process has loaded
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-o", so,
                    os.path.join(ROOT, "ginkgo_b200", "host", "capi.cpp")] + san + objs + link_args(), check=True)
    return api._configure_host_lib(ctypes.CDLL(so))
