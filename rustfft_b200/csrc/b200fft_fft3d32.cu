// libb200fft.so -- the f32 compiled axis pass of the 3-D plans (AxisKernel, fft3d.h), in a translation unit of its own.
#include "rt_cuda.h"
#define B2_PART_FFT3D32 1
#include "impl.inl"
