// TEST INFRASTRUCTURE ONLY -- tacotron_b200/csrc/gru.cu compiled for the host emulation (see emu.h)
#include "emu.h"
#include "../../tacotron_b200/csrc/gru.cu"
