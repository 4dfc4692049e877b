"""taco_highway_stack_fwd's descriptor: the ctypes mirror has the C layout, and descriptors the kernel cannot run are
refused on the host with a message, before any device call (no GPU needed)."""
import ctypes
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_desc_layout_matches_header():
    from tacotron_b200 import _lib
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "taco_b200.h"
int main(void){ printf("%zu %zu %zu %d\n", sizeof(taco_highway_stack_desc), offsetof(taco_highway_stack_desc, xp_p),
                       offsetof(taco_highway_stack_desc, impl), TACO_HIGHWAY_STACK_MAX); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c"); exe = os.path.join(d, "p")
        open(c, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        size, off_xp, off_impl, hmax = map(int, subprocess.check_output([exe]).split())
    D = _lib.HighwayStackDesc
    assert (ctypes.sizeof(D), D.xp_p.offset, D.impl.offset, _lib.HIGHWAY_STACK_MAX) == (size, off_xp, off_impl, hmax)


def _desc(C=128, L=4, impl=2):
    from tacotron_b200 import _lib
    d = _lib.HighwayStackDesc()
    d.X = 0x1000; d.ldx = C; d.M = 1000; d.C = C
    if C != 128:
        d.Wd_p = 0x2000; d.ldwd = (C + 31) // 32 * 32; d.bd = 0x3000
    d.L = L
    for l in range(min(L, _lib.HIGHWAY_STACK_MAX)):
        d.hw_p[l] = 0x10000 * (l + 1); d.hw_b[l] = 0x10000 * (l + 1) + 0x800
    d.ldhw = 128
    d.xp_p = 0x100000; d.ldxp = 128; d.xp_b = 0x200000
    d.Y = 0x300000; d.ldy = 768
    d.impl = impl
    return d


@pytest.mark.parametrize("change,msg", [
    (dict(impl=0), "TACO_IMPL_TC3"),
    (dict(C=200), "bad sizes"),
    (dict(L=5), "highway layers"),
    (dict(L=0), "highway layers"),
])
def test_refused_descriptors(change, msg):
    from tacotron_b200 import _lib
    d = _desc(**change)
    rc = _lib.lib().taco_highway_stack_fwd(ctypes.byref(d), None)
    assert rc != 0
    assert msg in _lib.lib().taco_last_error().decode()


def test_refused_fields():
    from tacotron_b200 import _lib
    lib = _lib.lib()
    d = _desc(C=128); d.Wd_p = 0x2000                         # a width-fixing dense with 128-wide inputs
    assert lib.taco_highway_stack_fwd(ctypes.byref(d), None) != 0 and b"iff C != 128" in lib.taco_last_error()
    d = _desc(C=80); d.ldy = 700
    assert lib.taco_highway_stack_fwd(ctypes.byref(d), None) != 0 and b"ldy" in lib.taco_last_error()
    d = _desc(C=80); d.X = 0x1004                             # TMA needs 16-byte aligned rows
    assert lib.taco_highway_stack_fwd(ctypes.byref(d), None) != 0 and b"16-byte aligned" in lib.taco_last_error()
