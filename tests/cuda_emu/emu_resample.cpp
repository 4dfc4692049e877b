// TEST INFRASTRUCTURE ONLY -- tacotron_b200/csrc/resample.cu compiled for the host emulation (see emu.h).
// The three round-to-nearest intrinsics of the kernel (one rounding per operation, no contraction) are plain double
// arithmetic on the host: g++ does not contract across statements in ISO C++ mode.
#include "emu.h"
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline float __double2float_rn(double a) { return (float)a; }
#include "../../tacotron_b200/csrc/resample.cu"
