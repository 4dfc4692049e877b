// TEST INFRASTRUCTURE ONLY -- tacotron_b200/csrc/features.cu compiled for the host emulation (see emu.h).
// The two round-to-nearest intrinsics the pre-emphasis uses (one rounding per operation, no contraction) are plain
// float arithmetic on the host: g++ does not contract across statements in ISO C++ mode.
#include "emu.h"
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fsub_rn(float a, float b) { return a - b; }
#include "../../tacotron_b200/csrc/features.cu"
