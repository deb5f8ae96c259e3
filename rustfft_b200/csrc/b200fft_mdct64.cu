// libb200fft.so -- the f64 MDCT kernels (MdctKernel, MdctFoldKernel, ImdctOlaKernel; mdct.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_MDCT64 1
#include "impl.inl"
