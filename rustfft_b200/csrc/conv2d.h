// 2-D FFT convolution of real images with one real filter (b200fft_conv2d_*): a circular convolution of P x Q, Q = 2 M, large
// enough that the requested output rows and columns are free of aliasing, in three passes over half-size complex data:
//   row pass      Conv2dRowKernel<T, 0>   image row [W] reals, read as z[m] = x[2m] + i x[2m+1] (0 past W) --FFT_M--> Z [H][M]
//   column pass   Conv2dColumnKernel<T>   column k = 0 .. M of the row spectra (real.h's unpack on the load, rows e >= H zero)
//                                         --FFT_P--> x G[k1][k], conj --FFT_P--> conj: rows r0 .. r0 + Ho - 1 --> Y [Ho][M + 1]
//   inverse rows  Conv2dRowKernel<T, 1>   row of Y, real.h's pack on the load --IFFT_M--> reals c0 .. c0 + Wo - 1 --> out [Wo]
// G = rfft2(h wrapped onto P x Q) / (P Q), so the three unnormalised passes give plain sums.  Every FFT has a run-time radix list
// of 2, 3, 4, 5, 7, 8, 16 (P and M are 7-smooth); each stage is one phase / step over a ping-pong pair of shared-memory buffers,
// as in SmoothKernel and SmoothConvKernel (kernels.h).
#pragma once
#include "kernels.h"

namespace b2 {

// scalar real loads and stores of the images (an odd width puts rows at odd offsets): streamed, read or written once
template <typename T> B2_HD T ld_real_cs(const T* p) {
#if defined(__CUDA_ARCH__)
    return __ldcs(p);
#else
    return *p;
#endif
}
template <typename T> B2_HD void st_real_cs(T* p, T v) {
#if defined(__CUDA_ARCH__)
    __stcs(p, v);
#else
    *p = v;
#endif
}

// ------------------------------------------------------------------------------------------
// Conv2dRowKernel: one M-point FFT per row, F rows per CTA (SmoothKernel's stage loop and index algebra).
//   DIR 0 (forward): row g = (image, row) of the real images, W reals each -> Z[g][0 .. M - 1]
//   DIR 1 (inverse): row g of Y [rows][M + 1]: z'[k] = A + i conj(W_Q^k) B, A / B = Y[k] +/- conj Y[M - k] (real.h's pack, no
//                    row reflection: the column inverse is already done), inverse FFT_M (re/im swapped on load and store), and
//                    the reals c0 .. c0 + Wo - 1 of z' go to out[g][0 .. Wo - 1]
// ------------------------------------------------------------------------------------------
template <typename T, int DIR>
struct Conv2dRowKernel {
    using T_ = T;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 3;
    static constexpr int MAX_STAGES = 8;
    static constexpr int NPHASE = MAX_STAGES;
    static constexpr size_t SMEM_BYTES = 0;  // run-time sized: Params::smem_bytes
    struct Params {
        const void* in;    // DIR 0: T [rows][width];          DIR 1: cx<T> [rows][M + 1]
        void* out;         // DIR 0: cx<T> [rows][M];          DIR 1: T [rows][width]
        const cx<T>* tw;   // packed stage twiddles of the M-point FFT (layout as in SmoothKernel)
        const cx<T>* wk;   // DIR 1: W_Q^k, k = 0 .. M - 1
        uint64_t n_fft;    // rows of this launch
        uint32_t n;        // M
        uint32_t width;    // DIR 0: W, reals per image row;   DIR 1: Wo, reals per output row
        uint32_t c0;       // DIR 1: first real of z' that is stored
        uint32_t n_stages, f_per_cta, smem_bytes;
        uint32_t radix[MAX_STAGES];
        uint32_t tw_off[MAX_STAGES];
        FastDiv div_t[MAX_STAGES];  // by T_s = M / radix[s]
        FastDiv div_p[MAX_STAGES];  // by p_s = product of the radices before s
    };
    struct Regs {};

    template <int R>
    static B2_HD void stage(const Params& p, uint32_t bid, int tid, int s, cx<T>* smem) {
        const uint32_t n = p.n, F = p.f_per_cta;
        const uint32_t pp = p.div_p[s].d, T_s = p.div_t[s].d;
        const bool first = (s == 0), last = (s == (int)p.n_stages - 1);
        const cx<T>* src_buf = smem + (size_t)((s + 1) & 1) * F * n;
        cx<T>* dst_buf = smem + (size_t)(s & 1) * F * n;
        const cx<T>* tws = p.tw + p.tw_off[s];
        for (uint32_t b = (uint32_t)tid; b < F * T_s; b += NT) {
            const uint32_t f = p.div_t[s].div(b), i = b - f * T_s;
            const uint64_t g = (uint64_t)bid * F + f;
            if (g >= p.n_fft) continue;
            const uint32_t k = i - p.div_p[s].div(i) * pp;
            cx<T> a[R];
            if (first) {
                if constexpr (DIR == 0) {
                    const T* src = (const T*)p.in + g * p.width;
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) {
                        const uint32_t j = 2 * (i + (uint32_t)q * T_s);
                        a[q] = mk<T>(j < p.width ? ld_real_cs(src + j) : (T)0, j + 1 < p.width ? ld_real_cs(src + j + 1) : (T)0);
                    }
                } else {
                    const cx<T>* src = (const cx<T>*)p.in + g * (n + 1);
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) {
                        const uint32_t kk = i + (uint32_t)q * T_s;
                        const cx<T> yk = ld_cs(src + kk), ym = conj(ld_cs(src + (n - kk)));
                        const cx<T> t = cmulc(yk - ym, ldg(p.wk + kk));  // conj(W^k) B
                        a[q] = swap_ri(yk + ym + mk<T>(-t.y, t.x));      // A + i conj(W^k) B, swapped for the inverse FFT
                    }
                }
            } else {
                const cx<T>* src = src_buf + (size_t)f * n + i;
                B2_UNROLL
                for (int q = 0; q < R; ++q) a[q] = src[(size_t)q * T_s];
                B2_UNROLL
                for (int q = 1; q < R; ++q) a[q] = cmul(a[q], ldg(tws + (size_t)(q - 1) * pp + k));
            }
            Bfly<R, T>::run(a);
            const uint32_t base = (i - k) * R + k;
            if (last) {
                if constexpr (DIR == 0) {
                    cx<T>* dst = (cx<T>*)p.out + g * n + base;  // re-read by the column pass
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) dst[(size_t)m * pp] = a[m];
                } else {
                    T* dst = (T*)p.out + g * p.width;
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) {
                        const cx<T> v = swap_ri(a[m]);
                        const uint32_t j = 2 * (base + (uint32_t)m * pp) - p.c0;  // (wraps to a large value below c0)
                        if (j < p.width) st_real_cs(dst + j, v.x);
                        if (j + 1 < p.width) st_real_cs(dst + (j + 1), v.y);
                    }
                }
            } else {
                cx<T>* dst = dst_buf + (size_t)f * n + base;
                B2_UNROLL
                for (int m = 0; m < R; ++m) dst[(size_t)m * pp] = a[m];
            }
        }
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>* smem) {
        if (P >= (int)p.n_stages) return;
        switch (p.radix[P]) {  // 7-smooth lengths: no prime butterflies above 7
            case 2: stage<2>(p, bid, tid, P, smem); break;
            case 3: stage<3>(p, bid, tid, P, smem); break;
            case 4: stage<4>(p, bid, tid, P, smem); break;
            case 5: stage<5>(p, bid, tid, P, smem); break;
            case 7: stage<7>(p, bid, tid, P, smem); break;
            case 8: stage<8>(p, bid, tid, P, smem); break;
            case 16: stage<16>(p, bid, tid, P, smem); break;
            default: break;
        }
    }
};

// ------------------------------------------------------------------------------------------
// Conv2dColumnKernel: the M + 1 spectrum columns k of every image, F columns per CTA, one P-point forward FFT, the pointwise
// product with the filter's spectrum, one P-point inverse FFT (SmoothConvKernel's 2 S steps, the step index run-time data):
//   step 0       column k of the row spectra, rows e < H: E + W_Q^k O, E / O from Z[e][k mod M] and conj Z[e][(M - k) mod M]
//                (real.h's unpack), rows e >= H: 0
//   step S       times G[k1][k] and conjugated on the load (the inverse FFT as conj(FFT(conj)))
//   step 2S - 1  conjugated; only rows r0 .. r0 + Ho - 1 are stored, to Y[r - r0][k]
// CTA bid takes column group bid / images of image bid mod images: consecutive CTAs read the same F columns of G for successive
// images, so G (P (M + 1) entries, read through the table path) comes from L2 rather than HBM.  Threads: column fastest (the F
// columns of a row are adjacent in Z, G and Y); shared memory [element][column].
// ------------------------------------------------------------------------------------------
template <typename T>
struct Conv2dColumnKernel {
    using T_ = T;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 3;
    static constexpr int MAX_STAGES = 8;
    static constexpr size_t SMEM_BYTES = 0;  // run-time sized: Params::smem_bytes
    struct Params {
        const cx<T>* in;    // Z [images][H][M]
        cx<T>* out;         // Y [images][Ho][M + 1]
        const cx<T>* tw;    // packed stage twiddles of the P-point FFT (layout as in SmoothKernel)
        const cx<T>* wk;    // W_Q^k, k = 0 .. M
        const cx<T>* g;     // G [P][M + 1]
        uint32_t n;         // P
        uint32_t half_w;    // M
        uint32_t h;         // H: rows of Z per image
        uint32_t r0, ho;    // first stored row, rows stored
        uint32_t n_img;     // images of this launch
        uint32_t n_stages, f_per_cta, smem_bytes;
        uint32_t radix[MAX_STAGES];
        uint32_t tw_off[MAX_STAGES];
        FastDiv div_t[MAX_STAGES];  // by T_s = P / radix[s]
        FastDiv div_p[MAX_STAGES];  // by p_s = product of the radices before s
        FastDiv div_f, div_img;
    };

    template <int R>
    static B2_HD void stage(const Params& p, uint32_t bid, int tid, uint32_t step, cx<T>* smem) {
        const uint32_t S = p.n_stages, P = p.n, F = p.f_per_cta, M = p.half_w;
        const bool second = step >= S;
        const uint32_t s = second ? step - S : step;
        const bool first_s = (s == 0), last_s = (s == S - 1);
        const uint32_t pp = p.div_p[s].d, T_s = p.div_t[s].d;
        const cx<T>* src_buf = smem + (size_t)((step + 1) & 1) * F * P;
        cx<T>* dst_buf = smem + (size_t)(step & 1) * F * P;
        const cx<T>* tws = p.tw + p.tw_off[s];
        const uint32_t grp = p.div_img.div(bid), b = bid - grp * p.n_img;  // column group, image
        for (uint32_t idx = (uint32_t)tid; idx < F * T_s; idx += NT) {
            const uint32_t i = p.div_f.div(idx), f = idx - i * F;
            const uint32_t col = grp * F + f;
            if (col > M) continue;
            const uint32_t k = i - p.div_p[s].div(i) * pp;
            cx<T> a[R];
            if (first_s && !second) {
                const cx<T>* src = p.in + (uint64_t)b * p.h * M;
                const uint32_t ka = col == M ? 0u : col, kb = col == 0 ? 0u : M - col;
                const cx<T> w = ldg(p.wk + col);
                const T half = (T)0.5;
                B2_UNROLL
                for (int q = 0; q < R; ++q) {
                    const uint32_t e = i + (uint32_t)q * T_s;
                    if (e < p.h) {
                        const cx<T>* row = src + (uint64_t)e * M;
                        const cx<T> zk = ldg_stream(row + ka), zm = conj(ldg_stream(row + kb));
                        const cx<T> ev = mk<T>((zk.x + zm.x) * half, (zk.y + zm.y) * half);
                        const cx<T> d = mk<T>((zk.x - zm.x) * half, (zk.y - zm.y) * half);  // = i O
                        a[q] = ev + cmul(mk<T>(d.y, -d.x), w);                              // E + W^k O
                    } else {
                        a[q] = mk<T>(0, 0);
                    }
                }
            } else {
                B2_UNROLL
                for (int q = 0; q < R; ++q) a[q] = src_buf[(size_t)(i + (uint32_t)q * T_s) * F + f];
                if (first_s) {  // first stage of the inverse FFT: times the filter's spectrum, conjugated
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) a[q] = conj(cmul(a[q], ldg(p.g + (size_t)(i + (uint32_t)q * T_s) * (M + 1) + col)));
                } else {
                    B2_UNROLL
                    for (int q = 1; q < R; ++q) a[q] = cmul(a[q], ldg(tws + (size_t)(q - 1) * pp + k));
                }
            }
            Bfly<R, T>::run(a);
            const uint32_t base = (i - k) * R + k;
            if (last_s && second) {
                cx<T>* dst = p.out + (uint64_t)b * p.ho * (M + 1) + col;
                B2_UNROLL
                for (int m = 0; m < R; ++m) {
                    const uint32_t r = base + (uint32_t)m * pp - p.r0;  // (wraps to a large value below r0)
                    if (r < p.ho) dst[(uint64_t)r * (M + 1)] = conj(a[m]);
                }
            } else {
                B2_UNROLL
                for (int m = 0; m < R; ++m) dst_buf[(size_t)(base + (uint32_t)m * pp) * F + f] = a[m];
            }
        }
    }

    static B2_HD void step(const Params& p, uint32_t bid, int tid, uint32_t st, cx<T>* smem) {
        if (st >= 2 * p.n_stages) return;
        const uint32_t s = st >= p.n_stages ? st - p.n_stages : st;
        switch (p.radix[s]) {
            case 2: stage<2>(p, bid, tid, st, smem); break;
            case 3: stage<3>(p, bid, tid, st, smem); break;
            case 4: stage<4>(p, bid, tid, st, smem); break;
            case 5: stage<5>(p, bid, tid, st, smem); break;
            case 7: stage<7>(p, bid, tid, st, smem); break;
            case 8: stage<8>(p, bid, tid, st, smem); break;
            case 16: stage<16>(p, bid, tid, st, smem); break;
            default: break;
        }
    }
};


}  // namespace b2
