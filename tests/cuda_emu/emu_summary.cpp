// TEST INFRASTRUCTURE ONLY -- tacotron_b200/csrc/summary.cu compiled for the host emulation (see emu.h).
// The kernel's shared-memory histogram counts with the 32-bit integer atomicAdd, which emu.h does not define.
#include "emu.h"
inline unsigned atomicAdd(unsigned* p, unsigned v) { return std::atomic_ref<unsigned>(*p).fetch_add(v, std::memory_order_relaxed); }
using std::isfinite;
#include "../../tacotron_b200/csrc/summary.cu"
