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
//
// LAYOUT selects which filter a block multiplies by and which rows it reads and writes (C filters, output row (b, c) at
// (b C + c) out_len):
//   CONV_ONE          one filter for every row: the single-filter plans (OverlapSaveKernel below).
//   CONV_PER_CHANNEL  input row (b, c) at (b C + c) n, filtered by h_c.  Loads and stores as CONV_ONE over batch C rows.
//                     Complex: row g uses the spectrum H + (g mod C) M.  REAL: rows 2u and 2u + 1 (channels c_a = 2u mod C,
//                     c_b = c_a + 1 mod C; for odd C a pair wraps into the next batch element) share one block z = a + i b
//                     but not their filter.  With A, B the spectra of the real blocks, conj Z[M-k] = A[k] - i B[k], so
//                         W[k] = P[k] Z[k] + Q[k] conj Z[M-k] = A H_a + i B H_b,   P = (H_a + H_b) / 2,  Q = (H_a - H_b) / 2
//                     and the inverse returns a (*) h_a + i (b (*) h_b).  Z[M-k] lives in another thread's registers: the last
//                     forward phase writes Z to shared memory, the next phase reads the mirror and forms W, and the second FFT
//                     starts one phase later (its stage 0 overwrites the buffer).  The (P, Q) tables ([2][M] each) are indexed
//                     by u mod C' (C' = C / 2 for even C, else C; slot s holds the pair c_a = 2 s mod C).
//   CONV_SHARED       input row b (batch rows), filtered by every h_c.  Blocks are numbered (b, block j, slot s) with s
//                     fastest, so the blocks that read one input span run back to back and read it from L2.  Complex: slot s =
//                     channel c, spectrum H + c M.  REAL: slot s = channel pair (2s, 2s + 1): z = x_b (imaginary part zero)
//                     times G_s = H_2s + i H_2s+1 (H_C = 0 for odd C) gives x (*) h_2s + i (x (*) h_2s+1), stored to the
//                     two channels (the second only if it exists).
// The channel layouts number a launch's blocks from a (unit or batch element, block, slot) start and find a block's slot with one
// more 32-bit division by the slot period (C, C' or ceil(C / 2)).
#pragma once
#include <algorithm>
#include <type_traits>

#include "kernels.h"

namespace b2 {

enum { CONV_ONE = 0, CONV_PER_CHANNEL = 1, CONV_SHARED = 2 };

template <class G, bool REAL, int MINB = 1, int LAYOUT = CONV_ONE>
struct ChannelOverlapSaveKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = MINB;
    static constexpr int NP1 = Eng::NPHASE;
    static constexpr bool XCH = REAL && LAYOUT == CONV_PER_CHANNEL;  // Z[M-k] through shared memory between the two FFTs
    static constexpr int S2 = XCH ? NP1 + 1 : NP1 - 1;                  // phase of the second FFT's stage 0
    static constexpr int NPHASE = S2 + NP1;
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::SMEM_ELEMS;
    struct OneParams {
        const void* in;  // rows of n samples: cx<T>, or T when REAL
        void* out;       // rows of out_len samples, same type
        const cx<T>* H;  // M entries: FFT_M(h zero-padded to M) / M  (channel layouts: the tables above, M entries per row)
        const cx<T>* tw; // stage twiddles of the M-point FFT
        uint64_t n, out_len;
        int64_t shift;   // s0 - (m - 1): input index of element 0 of block 0
        uint64_t rows;   // rows in the batch (REAL: row 2u + 1 of the last unit may not exist)
        uint64_t r0;     // unit of the launch's first block (CONV_SHARED: batch element)
        uint64_t cnt;    // blocks in this launch
        uint32_t b0;     // block (within its unit) of the launch's first block
        uint32_t L, ov;  // valid outputs per block, m - 1
        FastDiv div_nblk;
    };
    struct ChannelParams : OneParams {
        uint32_t nch;    // C
        uint32_t c0;     // table slot of the launch's first block
        FastDiv div_per; // by the slot period
    };
    using Params = std::conditional_t<LAYOUT == CONV_ONE, OneParams, ChannelParams>;
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
    // channel layouts: the rows of FFT slot f (offsets in samples of its input and output rows), its table slot, and whether the
    // second real row of a REAL block exists on the load and on the store side
    struct Rows {
        uint64_t in, out;
        uint32_t s;
        bool b_in, b_out;
    };
    static B2_HD Rows rows_of(const Params& p, uint32_t bid, int f, uint64_t& t0, bool& ok) {
        Rows w;
        if constexpr (LAYOUT == CONV_SHARED) {
            const uint64_t g = (uint64_t)bid * G::F + f;
            ok = g < p.cnt;
            const uint32_t c = p.c0 + (uint32_t)(ok ? g : 0);
            const uint32_t q1 = p.div_per.div(c);
            const uint32_t jj = p.b0 + q1;
            const uint32_t q2 = p.div_nblk.div(jj);
            const uint64_t b = p.r0 + q2;
            t0 = (uint64_t)(jj - q2 * p.div_nblk.d) * p.L;
            w.s = c - q1 * p.div_per.d;
            const uint32_t ch = REAL ? 2 * w.s : w.s;
            w.in = b * p.n;
            w.out = (b * p.nch + ch) * p.out_len;
            w.b_in = false;
            w.b_out = ch + 1 < p.nch;
        } else {
            uint64_t unit;
            locate(p, bid, f, unit, t0, ok);
            w.in = (REAL ? 2 * unit : unit) * p.n;
            w.out = (REAL ? 2 * unit : unit) * p.out_len;
            w.b_in = w.b_out = 2 * unit + 1 < p.rows;
            const uint32_t c = p.c0 + (uint32_t)(unit - p.r0);
            w.s = c - p.div_per.div(c) * p.div_per.d;
        }
        return w;
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        if constexpr (P == 0) {
            uint64_t unit, t0;
            bool ok;
            Rows w{};
            if constexpr (LAYOUT == CONV_ONE) {
                locate(p, bid, f, unit, t0, ok);
            } else {
                w = rows_of(p, bid, f, t0, ok);
                unit = 0;
            }
            // element e of the block is input sample base + e: valid for e in [e_lo, e_hi) (32-bit compares per element, one 64-bit
            // base pointer per thread)
            const int64_t base = (int64_t)t0 + p.shift;
            const int32_t e_lo = (int32_t)(base < 0 ? -base : 0);
            const int32_t e_hi = !ok || base >= (int64_t)p.n ? 0 : (int32_t)std::min<int64_t>((int64_t)p.n - base, G::L);
            if constexpr (REAL) {
                const T* a = (const T*)p.in + (LAYOUT == CONV_ONE ? 2 * unit * p.n : w.in) + base;
                const bool has_b = LAYOUT == CONV_ONE ? 2 * unit + 1 < p.rows : w.b_in;
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
                const cx<T>* a = (const cx<T>*)p.in + (LAYOUT == CONV_ONE ? unit * p.n : w.in) + base;
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
        if constexpr (XCH && P == NP1 - 1) {
            // the last forward stage read no shared memory: Z goes there for the mirror reads of the next phase
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) smem[G::sidx(f, j + G::TP * q)] = r.v[q];
        }
        if constexpr (XCH && P == NP1) {
            // W[k] = P[k] Z[k] + Q[k] conj Z[M-k], conjugated for the second FFT
            uint64_t t0;
            bool ok;
            const cx<T>* tp = p.H + (size_t)rows_of(p, bid, f, t0, ok).s * (2 * G::L);
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                const cx<T> zm = conj(smem[G::sidx(f, (G::L - k) & (G::L - 1))]);
                r.v[q] = conj(cmul(r.v[q], ldg(tp + k)) + cmul(zm, ldg(tp + G::L + k)));
            }
        }
        if constexpr (P == S2) {
            // pointwise multiply + conjugate (XCH: done above), then stage 0 of the second FFT straight from registers
            if constexpr (LAYOUT == CONV_ONE) {
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) r.v[q] = conj(cmul(r.v[q], ldg(p.H + j + G::TP * q)));
            } else if constexpr (!XCH) {
                uint64_t t0;
                bool ok;
                const cx<T>* hp = p.H + (size_t)rows_of(p, bid, f, t0, ok).s * G::L;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) r.v[q] = conj(cmul(r.v[q], ldg(hp + j + G::TP * q)));
            }
            Eng::template phase<0>(tid, r.v, smem, p.tw);
        }
        if constexpr (P > S2) {
            Eng::template phase<P - S2>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NPHASE - 1) {
            uint64_t unit, t0;
            bool ok;
            Rows w{};
            if constexpr (LAYOUT == CONV_ONE) {
                locate(p, bid, f, unit, t0, ok);
            } else {
                w = rows_of(p, bid, f, t0, ok);
                unit = 0;
            }
            // element e >= m - 1 is output t0 + e - (m - 1): stored for e in [ov, e_hi)
            const uint64_t left = p.out_len - t0 + p.ov;  // (t0 < out_len for every block of a launch)
            const int32_t e_hi = ok ? (int32_t)std::min<uint64_t>(left, G::L) : 0;
            const int32_t ov = (int32_t)p.ov;
            if constexpr (REAL) {
                T* a = (T*)p.out + (LAYOUT == CONV_ONE ? 2 * unit * p.out_len : w.out) + ((int64_t)t0 - ov);
                const bool has_b = LAYOUT == CONV_ONE ? 2 * unit + 1 < p.rows : w.b_out;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    if (e >= ov && e < e_hi) {
                        st_stream_r(a + e, r.v[q].x);
                        if (has_b) st_stream_r(a + p.out_len + e, -r.v[q].y);
                    }
                }
            } else {
                cx<T>* a = (cx<T>*)p.out + (LAYOUT == CONV_ONE ? unit * p.out_len : w.out) + ((int64_t)t0 - ov);
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int32_t e = j + G::TP * q;
                    if (e >= ov && e < e_hi) st_stream(a + e, conj(r.v[q]));
                }
            }
        }
    }
};

// The single-filter plans' kernel: a type of its own (not an alias), so that its instantiations keep their symbol names.
template <class G, bool REAL, int MINB = 1>
struct OverlapSaveKernel : ChannelOverlapSaveKernel<G, REAL, MINB, CONV_ONE> {};

}  // namespace b2
