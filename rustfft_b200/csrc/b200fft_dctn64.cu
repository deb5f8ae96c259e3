// libb200fft.so -- the f64 column kernels of the 2-D / 3-D DCTs and DSTs (DctAxisKernel, DctTransposeKernel; dct.h), in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_DCTN64 1
#include "impl.inl"
