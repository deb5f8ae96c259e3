// libb200fft.so -- the f32 column passes of the 2-D real transforms (Real2dColumnKernel, kernels.h), in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_REAL2D32 1
#include "impl.inl"
