// emu_lib.cpp -- TEST INFRASTRUCTURE ONLY.  The library half of libtaco_emu.so: the error string and the launch counter
// the product's kernel sources (the other emu_*.cpp units, one per .cu file) expect.  tests/emulator.py compiles all the
// units for the host over tests/cuda_emu/emu.h and links them into one library exporting the SAME C-ABI entry points;
// every test that takes its `emu` fixture drives them through ctypes with host pointers -- no GPU involved.
#include "emu.h"

#include <cstdarg>
#include <cstdio>

unsigned long long g_taco_launches = 0;
static thread_local char g_err[512];
void taco_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* taco_last_error(void) { return g_err; }

// the kernel sources are compiled as separate translation units (their anonymous-namespace helpers share names)
