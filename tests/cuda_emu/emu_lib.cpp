// emu_lib.cpp -- TEST INFRASTRUCTURE ONLY.  Builds libtaco_emu.so: the product's own kernel sources (audio.cu, data.cu,
// every kernel of train.cu) compiled with g++ over tests/cuda_emu/emu.h, exporting the SAME C-ABI entry points
// (taco_gemm, taco_set_gemm_impl, taco_bias_act, ..., taco_gl_*, taco_normalize_f16) so that tests/test_cuda_emu.py and
// tests/test_train_envelope_host.py can drive them through
// ctypes with host pointers and compare with the torch-CPU mirrors -- no GPU involved.
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

// the kernel sources are compiled as separate translation units (their anonymous-namespace helpers share names):
// emu_train.cpp, emu_audio.cpp, emu_data.cpp
