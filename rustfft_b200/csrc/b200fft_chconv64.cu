// libb200fft.so -- the f64 multi-channel overlap-save convolution kernels (conv.h, CONV_PER_CHANNEL / CONV_SHARED) and their plan
// builder, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_CHCONV64 1
#include "impl.inl"
