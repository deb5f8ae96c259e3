// libb200fft.so -- the f32 DCT / DST kernels (DctKernel, DctGenKernel; dct.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_DCT32 1
#include "impl.inl"
