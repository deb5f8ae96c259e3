// libb200fft.so -- the f64 passes of the 2-D convolution of real images (Conv2dRowKernel, Conv2dColumnKernel; conv2d.h), in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_CONV2D64 1
#include "impl.inl"
