// Modified DCTs of real rows (b200fft_mdct_*, rustdct's Mdct).  A plan fixes N (even), a real window w of 2N taps and the signal
// length L; a row x is padded as xp = N zeros, x, zeros up to (frames + 1) N samples, frames = ceil(L / N) + 1, and frame f is
// xp[f N, f N + 2N):
//     C[f][k] = sum_{n < 2N} w[n] xp[f N + n] cos(pi/N (n + 1/2 + N/2)(k + 1/2)),   k < N         (unnormalised; frame-major output)
//     y = crop_[N, N + L) of the overlap-add over f of (2/N) w[n] sum_k C[f][k] cos(pi/N (n + 1/2 + N/2)(k + 1/2)) at f N + n
// With z[n] = w[n] xp[f N + n] and h = N/2 the forward is the N-point DCT-IV (dct.h, = scipy.fft.dct(., 4) / 2) of the quarter fold
//     u[j] = -z[3h - 1 - j] - z[3h + j]   (j < h),        u[j] = z[j - h] - z[3h - 1 - j]   (j >= h)
// and the inverse unfolds u_f = DCT-IV(C[f]): sample p = j N + i of xp (i < N) is
//     (2/N) w[i] a_j[i] + (2/N) w[N + i] b_{j-1}[i],
//     a[i] = u[i + h] (i < h), -u[3h - 1 - i] (i >= h);      b[i] = -u[h - 1 - i] (i < h), -u[i - h] (i >= h)
// (DCT-IV is its own inverse up to N/2: the unscaled overlap-add of a Princen-Bradley window gives (N/2) x, hence the 2/N).
//
// MdctKernel<G>: the whole forward of N = 2M (M = G::L, a power of two) in one CTA pass, F frames per CTA.  Phase 0 forms u of the
// CTA's frames straight from the signal (two windowed samples per u value, zero outside [0, L)) into DctKernel's row layout; then
// DctKernel<G, DCT-IV>'s phases 1 .. NPHASE - 1 run unchanged, its store included.  The coefficient rows of a launch are contiguous
// across the batch, so a CTA may straddle two signal rows: each frame slot derives (row, f) from its global frame index.  One write
// of the coefficients; each signal sample is read by two frames (the second read expected from L1 / L2).
// MdctFoldKernel<T>: the general forward's fold, one thread per u value, into the output; the N-point DCT-IV plan then runs in place.
// ImdctOlaKernel<T>: the inverse's unfold and overlap-add after the N-point DCT-IV plan over every frame (into a workspace): one thread
// per output sample, which adds its two terms in a fixed order (no atomics: repeats are bit-identical).  The window table holds
// (2/N) w[n], evaluated in long double and rounded once.
#pragma once
#include "kernels.h"
#include "dct.h"

namespace b2 {

// read-only loads of the signal and the window (no output aliases them: the plans run out of place)
template <typename T> B2_HD T mdct_ld(const T* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// u[j] of the frame whose tap n sits at signal sample s0 + n (s0 = (f - 1) N: xp's N leading zeros make s0 = -N at f = 0)
template <typename T>
B2_HD T mdct_fold(const T* x, const T* w, int64_t s0, uint32_t L, uint32_t N, uint32_t j) {
    const uint32_t h = N / 2;
    auto z = [&](uint32_t n) {
        const int64_t s = s0 + n;
        return s >= 0 && s < (int64_t)L ? mdct_ld(w + n) * mdct_ld(x + s) : (T)0;
    };
    return j < h ? -z(3 * h - 1 - j) - z(3 * h + j) : z(j - h) - z(3 * h - 1 - j);
}

template <class G>
struct MdctKernel {
    using T = typename G::T;
    using DK = DctKernel<G, B200FFT_DCT4>;
    static constexpr int M = G::L, N = 2 * G::L, NT = G::NT;
    static constexpr int MIN_BLOCKS = DK::MIN_BLOCKS;
    static constexpr int NPHASE = DK::NPHASE;
    static constexpr size_t SMEM_BYTES = DK::SMEM_BYTES;
    struct Params {
        typename DK::Params dk;  // DctKernel's tables, out and rows (frames in this launch); its `in` is not used
        const T* in;             // the launch's first signal row
        const T* win;            // 2N taps
        uint32_t L;              // signal length
        FastDiv div_frames;      // by frames per row
    };
    using Regs = typename DK::Regs;

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        if constexpr (P == 0) {
            int f, j;
            tid_to_fj<G, JF>(tid, f, j);
            T* row = reinterpret_cast<T*>(smem) + f * N;  // DctKernel's layout: slot f at reals [f N, (f + 1) N)
            const uint64_t g = (uint64_t)bid * G::F + f;
            if (g < p.dk.rows) {
                const uint32_t rw = p.div_frames.div((uint32_t)g), fr = (uint32_t)g - rw * p.div_frames.d;
                const T* x = p.in + (uint64_t)rw * p.L;
                const int64_t s0 = ((int64_t)fr - 1) * N;
                B2_UNROLL
                for (int q = 0; q < 2 * G::E; ++q) row[j + G::TP * q] = mdct_fold(x, p.win, s0, p.L, (uint32_t)N, (uint32_t)(j + G::TP * q));
            } else {
                B2_UNROLL
                for (int q = 0; q < 2 * G::E; ++q) row[j + G::TP * q] = (T)0;
            }
        } else {
            DK::template phase<P>(p.dk, bid, tid, r, smem);
        }
    }
};

// general forward: u value i = g N + j of frame g of the launch (the launch starts at a row)
template <typename TT>
struct MdctFoldKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const T* in;        // the launch's first signal row
        T* out;             // [frames of the launch][N]
        const T* win;       // 2N taps
        uint64_t n_elem;    // frames of the launch * N (< 2^31)
        uint32_t L;
        FastDiv div_n;      // by N
        FastDiv div_frames; // by frames per row
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t N = p.div_n.d, g = p.div_n.div((uint32_t)i), j = (uint32_t)i - g * N;
        const uint32_t rw = p.div_frames.div(g), fr = g - rw * p.div_frames.d;
        p.out[i] = mdct_fold(p.in + (uint64_t)rw * p.L, p.win, ((int64_t)fr - 1) * N, p.L, N, j);
    }
};

// inverse: output sample t of row `row` of the launch from the DCT-IVs of its frames ([rows][frames][N])
template <typename TT>
struct ImdctOlaKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const T* in;       // u_f of the launch's rows
        T* out;            // rows of L samples
        const T* win;      // 2N taps (2/N) w[n]
        uint64_t n_elem;   // rows * L (< 2^31)
        uint32_t frames;
        FastDiv div_l;     // by L
        FastDiv div_n;     // by N
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t e = (uint64_t)bid * NT + tid;
        if (e >= p.n_elem) return;
        const uint32_t N = p.div_n.d, h = N / 2;
        const uint32_t row = p.div_l.div((uint32_t)e), t = (uint32_t)e - row * p.div_l.d;
        // xp sample t + N = j N + i: frame j's first half and frame j - 1's second half (1 <= j <= frames - 1)
        const uint32_t j = p.div_n.div(t) + 1, i = t + N - j * N;
        const T* u = p.in + ((uint64_t)row * p.frames + j) * N;  // u_j; u_{j-1} is N reals before it
        const T a = i < h ? u[i + h] : -u[3 * h - 1 - i];
        const T b = i < h ? -u[(int64_t)h - 1 - i - N] : -u[(int64_t)i - h - N];
        p.out[e] = mdct_ld(p.win + i) * a + mdct_ld(p.win + N + i) * b;
    }
};

}  // namespace b2
