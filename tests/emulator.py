"""The host emulation of the CUDA library (tests/cuda_emu): the product's own kernel sources compiled with g++ over
tests/cuda_emu/emu.h into one shared library, built at most once per test process and declared by the same table as
libtaco_b200.so (tacotron_b200/_lib.py SIGNATURES).

* `emu`: the module fixture the host tests take; skips when the CUDA toolkit headers are missing.
* `library()`: the library itself.
* `KernelsOver(lib)`: tacotron_b200.kernels running over `lib` -- the wrappers' own marshalling on CPU tensors, the
  NULL stream, and the device check accepting host memory.

The library's state (taco_set_gemm_impl) is shared by every module that uses it: a test that changes it restores it.
"""
import ctypes as C
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor
from contextlib import ExitStack
from unittest import mock

import pytest

from tacotron_b200 import _lib as L
from tacotron_b200 import kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
UNITS = ("emu_lib.cpp", "emu_train.cpp", "emu_audio.cpp", "emu_data.cpp", "emu_decoder_bwd.cpp", "emu_gru.cpp",
         "emu_gru_bwd.cpp", "emu_features.cpp", "emu_resample.cpp", "emu_summary.cpp")
_lib = None


def library():
    """the emulated library: the ten units compiled in parallel and linked once per process"""
    global _lib
    if _lib is not None:
        return _lib
    cuda_inc = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("CUDA toolkit headers not found")
    with tempfile.TemporaryDirectory(prefix="taco_emu_") as tmp:            # the loaded library outlives its file
        objs = [os.path.join(tmp, u.replace(".cpp", ".o")) for u in UNITS]

        def compile_unit(src, obj):
            subprocess.check_call(["g++", "-std=c++20", "-O1", "-fPIC", "-pthread", "-I", cuda_inc, "-I",
                                   os.path.join(ROOT, "include"), "-c", os.path.join(EMU, src), "-o", obj])
        with ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
            list(pool.map(compile_unit, UNITS, objs))
        out = os.path.join(tmp, "libtaco_emu.so")
        subprocess.check_call(["g++", "-shared", "-pthread", *objs, "-o", out])
        lib = C.CDLL(out)
    _lib = L.declare(lib, [n for n in L.EXPORTS if hasattr(lib, n)])
    return _lib


@pytest.fixture(scope="module")
def emu():
    return library()


class KernelsOver:
    """tacotron_b200.kernels over `lib`: each wrapper runs as the product runs it, with L.lib() -> lib, the NULL
    stream and host tensors accepted"""

    def __init__(self, lib):
        self.lib = lib

    def __getattr__(self, name):
        f = getattr(kernels, name)

        def call(*a, **kw):
            with ExitStack() as st:
                st.enter_context(mock.patch.object(L, "lib", lambda: self.lib))
                st.enter_context(mock.patch.object(kernels, "_st", lambda: None))
                st.enter_context(mock.patch.object(kernels, "_on_device", lambda t: True))
                return f(*a, **kw)
        return call
