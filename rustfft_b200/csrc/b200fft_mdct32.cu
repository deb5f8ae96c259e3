// libb200fft.so -- the f32 MDCT kernels (MdctKernel, MdctFoldKernel, ImdctOlaKernel; mdct.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_MDCT32 1
#include "impl.inl"
