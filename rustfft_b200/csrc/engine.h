// CTA-level Stockham autosort FFT engine.
//
// One CTA computes F independent FFTs of length L = R0*R1*...; every thread keeps E elements in
// registers (element slot q of thread j of an FFT is index j + (L/E)*q on the read side of EVERY
// stage and on the final output), performs E/R radix-R butterflies per stage and exchanges data
// through one padded shared-memory buffer between stages:
//
//   stage s, butterfly i in [0, L/R):  inputs  x[i + r*L/R]            r = 0..R-1
//                                      twiddle W_{pR}^{(i mod p) r}     p = R0*..*R(s-1)
//                                      outputs y[(i - i mod p)*R + (i mod p) + m*p]   m = 0..R-1
//
// (validated against numpy in tests/test_engine_model.py).  The same decomposition family as the
// reference's Radix4/RadixN (src/algorithm/radix4.rs:167-203, radixn.rs:250-333) -- a base FFT
// followed by layers of twiddled radix-r cross butterflies -- but auto-sorting, so there is no
// digit-reversal pass (src/array_utils.rs:372-437) and natural order falls out of the last stage.
//
// Shared-memory layout: sidx(f, e) = f*LP + e + (e >> 4).  The 1-in-16 pad makes the stride-R
// scatter of a stage conflict free for 8-byte accesses, the row pitch LP (see Geo) makes "f fastest"
// thread mappings (strided-column tiles) conflict free; see tests/test_engine_model.py.
#pragma once
#include "butterfly.h"
#include "common.h"

namespace b2 {

// largest power of two <= r (constant-folded inside unrolled loops)
B2_HD constexpr int hibit(int r) {
    int h = 1;
    while (2 * h <= r) h *= 2;
    return h;
}

B2_HD constexpr int ilog2_c(int r) {
    int l = 0;
    while ((1 << (l + 1)) <= r) ++l;
    return l;
}

enum Map { JF = 0, FF = 1 };  // which index varies fastest across consecutive threads

template <typename T_, int L_, int E_, int F_, typename RL_, int PS_ = 4>
struct Geo {
    using T = T_;
    using RL = RL_;
    static constexpr int L = L_, E = E_, F = F_, PS = PS_;
    static constexpr int TP = L / E;   // threads per FFT
    static constexpr int NT = F * TP;  // threads per CTA
    static constexpr int NS = RL::N;   // stages
    static constexpr int LPAD = L + (PS ? (L >> PS) : 0);
    // row pitch between the F FFTs of a CTA: a multiple of one 128-byte bank sweep plus UNIT/F elements
    // (plus 1 when F >= UNIT), so that the F (or UNIT) consecutive FFTs a transaction touches in the
    // "f fastest" mapping start on different bank groups -- tests/test_engine_model.py
    static constexpr int UNIT = 128 / (2 * (int)sizeof(T_));
    static constexpr int LPR = (LPAD + UNIT - 1) / UNIT * UNIT;
    static constexpr int LP = (F <= 1) ? LPAD : (F >= UNIT ? LPR + 1 : LPR + UNIT / F);
    static constexpr int SMEM_ELEMS = (NS > 1) ? F * LP : 0;
    static constexpr int TW_ELEMS = RL::tw_total();
    static constexpr bool POW2 = RL::all_pow2() && ((TP & (TP - 1)) == 0);
    static B2_HD int sidx(int f, int e) { return f * LP + e + (PS ? (e >> PS) : 0); }
    static_assert(RL::product() == L, "radices must multiply to L");
    static_assert(L % E == 0, "E must divide L");
};

template <class G, Map M>
B2_HD void tid_to_fj(int tid, int& f, int& j) {
    if (M == JF) {
        f = tid / G::TP;
        j = tid - f * G::TP;
    } else {
        j = tid / G::F;
        f = tid - j * G::F;
    }
}

template <class G, Map M0, Map M1>
struct Engine {
    using T = typename G::T;
    using RL = typename G::RL;
    static constexpr int E = G::E;

    // warm L1 with the table entries stage S loads per butterfly when the other factors are built as products (B2_TW_FEW):
    // W^(k 2^i) for thread (f, j) -- e.g. while the tile itself is still in flight
    template <int S>
    static B2_HD void prefetch_tw(int j, const cx<T>* tw) {
        constexpr int R = RL::get(S);
        constexpr int p = RL::product(S);
        constexpr int Q = E / R;
        B2_UNROLL
        for (int u = 0; u < Q; ++u) {
            const int i = j + u * G::TP;
            const int k = (p == 1) ? 0 : (i % p);
            const cx<T>* tp = tw + RL::tw_offset(S) + k;
            B2_UNROLL
            for (int r = 1; r < R; r <<= 1) prefetch_l1(tp + (r - 1) * p);
        }
    }

    // one stage: consumes v (slot q <-> element j + TP*q), produces either smem (not last) or v
    template <int S>
    static B2_HD void stage(int f, int j, cx<T> (&v)[E], cx<T>* smem, const cx<T>* tw) {
        constexpr int R = RL::get(S);
        constexpr int p = RL::product(S);
        constexpr int Q = E / R;
        constexpr bool last = (S == G::NS - 1);
        static_assert(E % R == 0, "every radix must divide E");
        cx<T> out[E];
        B2_UNROLL
        for (int u = 0; u < Q; ++u) {
            const int i = j + u * G::TP;
            const int k = (p == 1) ? 0 : (i % p);
            cx<T> a[R];
            B2_UNROLL
            for (int r = 0; r < R; ++r) a[r] = v[u + r * Q];
            if (S > 0) {
                const cx<T>* t = tw + RL::tw_offset(S) + k;
#if defined(B2_TW_FEW)
                if constexpr (R >= 8 && (R & (R - 1)) == 0 && sizeof(T) == 4) {
                    // load only W^(k 2^i) and build the other powers as products (each a product of at most
                    // log2 R correctly rounded table entries): log2 R loads instead of R - 1 through the LSU
                    cx<T> w[R];
                    B2_UNROLL
                    for (int r = 1; r < R; r <<= 1) w[r] = ldg(t + (r - 1) * p);
                    B2_UNROLL
                    for (int r = 3; r < R; ++r)
                        if (r & (r - 1)) {
                            const int hi = hibit(r);
                            w[r] = cmul(w[hi], w[r - hi]);
                        }
                    B2_UNROLL
                    for (int r = 1; r < R; ++r) a[r] = cmul(a[r], w[r]);
                } else
#endif
                {
                    B2_UNROLL
                    for (int r = 1; r < R; ++r) a[r] = cmul(a[r], ldg(t + (r - 1) * p));
                }
            }
            Bfly<R, T>::run(a);
            if (last) {
                B2_UNROLL
                for (int m = 0; m < R; ++m) out[u + m * Q] = a[m];
            } else {
                const int base = (i - k) * R + k;
                if constexpr (G::POW2) {
                    // pad(base + m p) == pad(base) + pad(m p) for power-of-two radices (k + m p never carries
                    // into bit 4 beyond what m p alone does): one address, compile-time offsets
                    cx<T>* wp = smem + G::sidx(f, base);
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) wp[m * p + (G::PS ? ((m * p) >> G::PS) : 0)] = a[m];
                } else {
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) smem[G::sidx(f, base + m * p)] = a[m];
                }
            }
        }
        if (last) {
            B2_UNROLL
            for (int q = 0; q < E; ++q) v[q] = out[q];
        }
    }

    template <int S>
    static B2_HD void read(int f, int j, cx<T> (&v)[E], const cx<T>* smem) {
        if constexpr (G::POW2) {
            // pad(j + TP q) == pad(j) + pad(TP q) when TP is a power of two: one address, constant offsets
            const cx<T>* rp = smem + G::sidx(f, j);
            B2_UNROLL
            for (int q = 0; q < E; ++q) v[q] = rp[G::TP * q + (G::PS ? ((G::TP * q) >> G::PS) : 0)];
        } else {
            B2_UNROLL
            for (int q = 0; q < E; ++q) v[q] = smem[G::sidx(f, j + G::TP * q)];
        }
    }

    // Phase numbering of one FFT:  0 = stage 0;  2s-1 = read inputs of stage s;  2s = stage s.
    static constexpr int NPHASE = 2 * G::NS - 1;

    // (f, j) owning the registers during phase P
    template <int P>
    static B2_HD void owner(int tid, int& f, int& j) {
        if (P == 0)
            tid_to_fj<G, M0>(tid, f, j);
        else
            tid_to_fj<G, M1>(tid, f, j);
    }
    // (f, j) owning the OUTPUT registers after the last phase
    static B2_HD void out_owner(int tid, int& f, int& j) { owner<NPHASE - 1>(tid, f, j); }

    template <int P>
    static B2_HD void phase(int tid, cx<T> (&v)[E], cx<T>* smem, const cx<T>* tw) {
        int f, j;
        owner<P>(tid, f, j);
        if constexpr (P == 0) {
            stage<0>(f, j, v, smem, tw);
        } else if constexpr (P % 2 == 1) {
            read<(P + 1) / 2>(f, j, v, smem);
        } else {
            stage<P / 2>(f, j, v, smem, tw);
        }
    }
};

}  // namespace b2
