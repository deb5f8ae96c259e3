// libb200fft.so -- the f32 short-time Fourier transform kernels (StftKernel, StftFrameKernel, IstftOlaKernel; stft.h) and their plan builders, in a translation unit of their own.
#include "rt_cuda.h"
#define B2_PART_STFT32 1
#include "impl.inl"
