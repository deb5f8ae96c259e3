// libb200fft.so -- the f64 analytic-signal kernels (HilbertKernel, HilbertMidKernel, HilbertPostKernel, HilbertPromoteKernel, HilbertSignKernel, HilbertRealKernel; hilbert.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_HILBERT64 1
#include "impl.inl"
