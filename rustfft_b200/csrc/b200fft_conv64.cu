// libb200fft.so -- the f64 overlap-save convolution kernels (conv.h) and their plan builder, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_CONV64 1
#include "impl.inl"
