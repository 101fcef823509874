// Translation unit of the split-operand ("bf16x3") instantiations of the wgmma conv kernels: the kernel templates
// are those of conv_tc.cu, compiled here with X3 = true (see conv_tc_dispatch_x3 there).
#define RAVE_TC_X3_UNIT 1
#include "conv_tc.cu"
