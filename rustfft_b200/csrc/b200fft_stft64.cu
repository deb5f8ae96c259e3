// libb200fft.so -- the f64 short-time Fourier transform kernels (StftKernel, StftFrameKernel, IstftOlaKernel; stft.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_STFT64 1
#include "impl.inl"
