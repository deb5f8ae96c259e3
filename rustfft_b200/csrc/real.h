// Real-input / real-output wrappers over the complex plans (SURVEY 8(f).4: the `realfft` ecosystem crate sits on RustFFT's Fft trait the
// same way; RustFFT itself has no real transform).  A real signal of even length N is read as M = N / 2 complex numbers
// z[m] = x[2m] + i x[2m+1] (the same bytes), transformed by the M-point complex plan, and unpacked:
//     E[k] = (Z[k] + conj Z[M-k]) / 2,   O[k] = (Z[k] - conj Z[M-k]) / (2i)        (FFTs of the even / odd samples)
//     X[k] = E[k] + W_N^k O[k],          X[M-k] = conj(E[k] - W_N^k O[k]),          k = 0 .. M/2   (X has M + 1 entries)
// The inverse packs the M + 1 spectrum entries back (scaled by 2, so that c2r(r2c(x)) = N x -- unnormalised like everything else here
// and like the realfft crate) and runs the M-point inverse plan straight into the real output.  Like numpy.fft.irfft it reads only
// the real parts of X[0] and X[M]: their imaginary parts have no real signal to belong to.
// One elementwise pass each, one thread per pair (k, M - k).
#pragma once
#include "kernels.h"

namespace b2 {

template <typename TT, int DIR>  // DIR 0: unpack after the forward FFT (r2c);  1: pack before the inverse FFT (c2r)
struct RealPackKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const cx<T>* in;   // DIR 0: Z, M per transform;        DIR 1: X, M + 1 per transform
        cx<T>* out;        // DIR 0: X, M + 1 per transform;    DIR 1: Z', M per transform
        const cx<T>* tw;   // W_N^k, k = 0 .. M/2
        uint64_t n_pairs;  // batch * (M/2 + 1)
        uint32_t M;
        FastDiv div_h;     // by M/2 + 1
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_pairs) return;
        const uint32_t h = p.div_h.d, M = p.M;
        const uint32_t b = p.div_h.div((uint32_t)i), k = (uint32_t)i - b * h, km = M - k;
        const cx<T> w = ldg(p.tw + k);
        const T half = (T)0.5;
        if (DIR == 0) {
            const cx<T>* z = p.in + (uint64_t)b * M;
            cx<T>* x = p.out + (uint64_t)b * (M + 1);
            const cx<T> zk = z[k], zm = conj(z[k == 0 ? 0 : km]);
            const cx<T> e = mk<T>((zk.x + zm.x) * half, (zk.y + zm.y) * half);
            const cx<T> d = mk<T>((zk.x - zm.x) * half, (zk.y - zm.y) * half);  // = i O
            const cx<T> o = mk<T>(d.y, -d.x);                                     // O = d / i
            const cx<T> wo = cmul(o, w);
            x[k] = e + wo;
            if (km != k) x[km] = conj(e - wo);
        } else {
            const cx<T>* x = p.in + (uint64_t)b * (M + 1);
            cx<T>* z = p.out + (uint64_t)b * M;
            cx<T> xk = x[k], xm = conj(x[km]);
            if (k == 0) {  // numpy's irfft: a real output has no room for Im X[0] or Im X[M], so both are dropped
                xk.y = (T)0;
                xm.y = (T)0;
            }
            const cx<T> a = xk + xm, bb = xk - xm;
            const cx<T> t = cmul(bb, conj(w));   // conj(W^k) B
            const cx<T> it = mk<T>(-t.y, t.x);   // i conj(W^k) B
            z[k] = a + it;
            if (k != 0 && km != k) z[km] = conj(a - it);
        }
    }
};

}  // namespace b2
