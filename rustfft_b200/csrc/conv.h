// Overlap-save FFT convolution in one CTA pass per block (the shape of BluesteinKernel, kernels.h, with other loads and
// stores):
//
//   block j of row r:  s[e] = x[r][j L + shift + e]  (e < M; 0 outside [0, n))        shift = s0 - (m - 1)
//                      c = IFFT_M(FFT_M(s) .* FFT_M(h zero-padded))                   (circular: c[e] is a full
//                                                                                        convolution sum for e >= m - 1)
//                      y[r][j L + e - (m - 1)] = c[e]   for m - 1 <= e < M, clipped to the output length
//
// with L = M - m + 1 valid outputs per block and s0 the start of the mode's output inside the full convolution (full: 0,
// same: (m - 1) / 2, valid: m - 1).  H = FFT_M(h) / M is computed on the host in long double; the inverse FFT is
// conj(FFT(conj(.))), so the kernel runs the same forward engine twice from registers:
//   phase 0:        load the block (zero padded)          -> forward FFT phases
//   phase NP1 - 1:  .* H, conjugate, stage 0 of the second FFT
//   last phase:     conjugate, store the m - 1 .. M - 1 outputs
// REAL: two real rows ride in one complex block (x = x_2u + i x_2u+1).  h is real, so the real and imaginary parts of c are
// the two rows' outputs; the imaginary half of the last unit of an odd batch is zero and never stored.
//
// Blocks are numbered unit-major (unit = row, or pair of rows when REAL): block g of a launch is block (b0 + g) mod nblk of
// unit r0 + (b0 + g) / nblk, so a launch never needs a 64-bit division.  Input and output must not overlap: neighbouring
// blocks read each other's output ranges as their halo.
#pragma once
#include <algorithm>

#include "kernels.h"

namespace b2 {

template <class G, bool REAL, int MINB = 1>
struct OverlapSaveKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = MINB;
    static constexpr int NP1 = Eng::NPHASE;
    static constexpr int NPHASE = 2 * NP1 - 1;
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::SMEM_ELEMS;
    struct Params {
        const void* in;  // rows of n samples: cx<T>, or T when REAL
        void* out;       // rows of out_len samples, same type
        const cx<T>* H;  // M entries: FFT_M(h zero-padded to M) / M
        const cx<T>* tw; // stage twiddles of the M-point FFT
        uint64_t n, out_len;
        int64_t shift;   // s0 - (m - 1): input index of element 0 of block 0
        uint64_t rows;   // rows in the batch (REAL: row 2u + 1 of the last unit may not exist)
        uint64_t r0;     // unit of the launch's first block
        uint64_t cnt;    // blocks in this launch
        uint32_t b0;     // block (within its unit) of the launch's first block
        uint32_t L, ov;  // valid outputs per block, m - 1
        FastDiv div_nblk;
    };
    struct Regs { cx<T> v[G::E]; };

    // unit, output index of the block's first valid sample, and whether this FFT slot holds a block of the launch
    static B2_HD void locate(const Params& p, uint32_t bid, int f, uint64_t& unit, uint64_t& t0, bool& ok) {
        const uint64_t g = (uint64_t)bid * G::F + f;
        ok = g < p.cnt;
        const uint32_t t = p.b0 + (uint32_t)(ok ? g : 0);
        const uint32_t q = p.div_nblk.div(t);
        unit = p.r0 + q;
        t0 = (uint64_t)(t - q * p.div_nblk.d) * p.L;
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        if constexpr (P == 0) {
            uint64_t unit, t0;
            bool ok;
            locate(p, bid, f, unit, t0, ok);
            // element e of the block is input sample base + e: valid for e in [e_lo, e_hi) (32-bit compares per element, one 64-bit
            // base pointer per thread)
            const int64_t base = (int64_t)t0 + p.shift;
            const int32_t e_lo = (int32_t)(base < 0 ? -base : 0);
            const int32_t e_hi = !ok || base >= (int64_t)p.n ? 0 : (int32_t)std::min<int64_t>((int64_t)p.n - base, G::L);
            if constexpr (REAL) {
                const T* a = (const T*)p.in + 2 * unit * p.n + base;
                const bool has_b = 2 * unit + 1 < p.rows;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    cx<T> v = mk<T>(0, 0);
                    if (e >= e_lo && e < e_hi) {
                        v.x = ld_stream_r(a + e);
                        if (has_b) v.y = ld_stream_r(a + p.n + e);
                    }
                    r.v[q] = v;
                }
            } else {
                const cx<T>* a = (const cx<T>*)p.in + unit * p.n + base;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    r.v[q] = (e >= e_lo && e < e_hi) ? ld_stream(a + e) : mk<T>(0, 0);
                }
            }
        }
        if constexpr (P < NP1) {
            Eng::template phase<P>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NP1 - 1) {
            // pointwise multiply + conjugate, then stage 0 of the second FFT straight from registers
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) r.v[q] = conj(cmul(r.v[q], ldg(p.H + j + G::TP * q)));
            Eng::template phase<0>(tid, r.v, smem, p.tw);
        }
        if constexpr (P >= NP1) {
            Eng::template phase<P - NP1 + 1>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NPHASE - 1) {
            uint64_t unit, t0;
            bool ok;
            locate(p, bid, f, unit, t0, ok);
            // element e >= m - 1 is output t0 + e - (m - 1): stored for e in [ov, e_hi)
            const uint64_t left = p.out_len - t0 + p.ov;  // (t0 < out_len for every block of a launch)
            const int32_t e_hi = ok ? (int32_t)std::min<uint64_t>(left, G::L) : 0;
            const int32_t ov = (int32_t)p.ov;
            if constexpr (REAL) {
                T* a = (T*)p.out + 2 * unit * p.out_len + ((int64_t)t0 - ov);
                const bool has_b = 2 * unit + 1 < p.rows;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    if (e >= ov && e < e_hi) {
                        st_stream_r(a + e, r.v[q].x);
                        if (has_b) st_stream_r(a + p.out_len + e, -r.v[q].y);
                    }
                }
            } else {
                cx<T>* a = (cx<T>*)p.out + unit * p.out_len + ((int64_t)t0 - ov);
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    if (e >= ov && e < e_hi) st_stream(a + e, conj(r.v[q]));
                }
            }
        }
    }
};

}  // namespace b2
