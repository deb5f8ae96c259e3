// libb200fft.so -- the f64 chirp-z transform kernels (the REAL BluesteinKernel instantiations; CztPreKernel, CztMulKernel, CztPostKernel: czt.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_CZT64 1
#include "impl.inl"
