// libb200fft.so -- the f32 analytic-signal kernels (HilbertKernel, HilbertMidKernel, HilbertPostKernel, HilbertPromoteKernel, HilbertSignKernel, HilbertRealKernel; hilbert.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_HILBERT32 1
#include "impl.inl"
