// Analytic signals of real rows (b200fft_hilbert_*, scipy.signal.hilbert along the last axis).  For a row x of N reals the output
// is z = x + i y, y[n] = sum_m x[m] (2/N) sum_{0<k<N/2} sin(2 pi k (n - m) / N): ifft(fft(x) h), h = 1, 2, .., 2, (1 at N/2), 0, ...
// The real part is the input itself, copied bit for bit.
//
// Even N = 2M: the row as M complex pairs z[m] = x[2m] + i x[2m+1], Z = FFT_M(z), then for 0 < k < M
//     Z'[k] = (2/N) (i s_k Z[k] + c_k conj Z[M-k]),   s_k = sin(pi k / M),  c_k = cos(pi k / M),   Z'[0] = 0
// and the unnormalised inverse M-point FFT of Z' is y as pairs: y[2m] + i y[2m+1].  One table entry t_k = (2/N) W_N^-k =
// (2/N) (c_k + i s_k) per k, in long double, rounded once:  Z'[k] = i t_k.y Z[k] + t_k.x conj Z[M-k].
//
// HilbertKernel<G>: the whole transform of N = 2M points (M = G::L, a power of two) in one CTA pass; the G::F engine slots of a CTA
// hold F consecutive rows (the last CTA's idle slots transform zeros and store nothing).
//   load:     z as M pairs, slot q of thread j is pair j + TP q (the engine's own register order)
//   engine:   Z = FFT_M(z)
//   combine:  Z to shared memory; thread (f, j) forms conj Z'[k] for its own k from Z[k] and Z[M-k]
//   engine:   FFT_M(conj Z'), whose conjugate is the unnormalised inverse of Z'
//   store:    pair m = j + TP q of the inverse is (y[2m], y[2m+1]): the thread writes out[2m] = (x[2m], y[2m]) and
//             out[2m+1] = (x[2m+1], y[2m+1]), one contiguous run per warp; x is read again from global memory (the CTA loaded
//             those bytes a few microseconds before, so the second read is expected to hit L2; not measured) -- keeping it in
//             registers would add E complex values per thread to kernels already at the 128-register cap (f32 M = 16384, most f64
//             sizes), and shared memory has no room for it at f32 M = 16384; no A/B of the two forms has been timed
// One read of N reals and one write of N complex values; no workspace.
//
// The general paths, one thread per element, in launches of fewer than 2^31 threads (the caller's chunks of whole rows):
//   even N:  (the M-point forward plan: x as M pairs -> workspace)  HilbertMidKernel: Z' in place, one thread per pair (k, M-k)
//            (the M-point inverse plan, in place)  HilbertPostKernel: out[n] = (x[n], y[n])
//   odd N:   HilbertPromoteKernel: out = (x, 0)  (the N-point forward plan, in place)  HilbertSignKernel: bin k times sgn(k) / N,
//            sgn = +1 for 0 < k < N/2, -1 above, 0 at k = 0  (the N-point inverse plan, in place: (~0, y))
//            HilbertRealKernel: x into the real parts
#pragma once
#include "kernels.h"

namespace b2 {

template <class G>
struct HilbertKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int M = G::L, F = G::F, NT = G::NT;
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, 32);
    static constexpr int P_Z = Eng::NPHASE - 1;         // the forward run's last phase, then Z to shared memory
    static constexpr int P_INV = P_Z + 2;               // first phase of the second run (after the combine)
    static constexpr int NPHASE = P_INV + Eng::NPHASE;  // the second run's last phase also stores
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::F * G::LP;
    static_assert((M & (M - 1)) == 0 && M >= 2, "M must be a power of two");
    static_assert(G::LP >= M, "a row's M bins must fit its slot of the engine's buffer");
    struct Params {
        const T* in;      // rows of N = 2M reals, at an even element
        cx<T>* out;       // rows of N complex values
        const cx<T>* tab; // t_k = (2/N) W_N^-k, k < M
        const cx<T>* tw;  // stage twiddles of the M-point FFT
        uint32_t rows;    // rows in this launch
    };
    struct Regs { cx<T> v[G::E]; };

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        const uint32_t row = bid * F + f;
        if constexpr (P == 0) {
            const cx<T>* x = reinterpret_cast<const cx<T>*>(p.in) + (size_t)row * M;
            // (a plain load: the store phase reads these bytes again, so they should stay in L2)
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) r.v[q] = row < p.rows ? x[j + G::TP * q] : mk<T>(0, 0);
        }
        if constexpr (P <= P_Z) Eng::template phase<P>(tid, r.v, smem, p.tw);
        if constexpr (P == P_Z) {
            // the engine's last phase reads no shared memory
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) smem[f * M + j + G::TP * q] = r.v[q];
        }
        if constexpr (P == P_Z + 1) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                if (q == 0 && j == 0) {
                    r.v[q] = mk<T>(0, 0);
                } else {
                    // conj Z'[k] = t.x Z[M-k] - i t.y conj Z[k]
                    const cx<T> zk = smem[f * M + k], zm = smem[f * M + M - k], t = ldg(p.tab + k);
                    r.v[q] = mk<T>(t.x * zm.x - t.y * zk.y, t.x * zm.y - t.y * zk.x);
                }
            }
        }
        if constexpr (P >= P_INV) Eng::template phase<P - P_INV>(tid, r.v, smem, p.tw);
        if constexpr (P == NPHASE - 1) {
            if (row >= p.rows) return;
            const cx<T>* x = reinterpret_cast<const cx<T>*>(p.in) + (size_t)row * M;
            cx<T>* o = p.out + (size_t)row * 2 * M;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int m = j + G::TP * q;
                const cx<T> xp = ld_stream(x + m);
                // (y[2m], y[2m+1]) = conj of the second run's output
                st_stream(o + 2 * m, mk<T>(xp.x, r.v[q].x));
                st_stream(o + 2 * m + 1, mk<T>(xp.y, -r.v[q].y));
            }
        }
    }
};

// the parameters every general-path pass takes (each uses the fields its comment names)
template <typename T>
struct HilbertPassParams {
    const T* x;         // input rows of N reals (Post, Promote, Real)
    cx<T>* w;           // workspace rows of M (Mid, Post) or output rows of N (Promote, Sign, Real)
    cx<T>* out;         // output rows of N (Post)
    const cx<T>* tab;   // t_k, k <= M/2 (Mid)
    T inv_n;            // (T) (1/N) (Sign)
    uint32_t len;       // M (Mid), N (Sign)
    FastDiv div;        // by M/2 + 1 (Mid), by N (Sign)
    uint64_t n_elem;    // threads of the launch
};

// workspace rows of Z (M bins) -> Z' in place: thread (row, k), k <= M/2, writes Z'[k] and Z'[M-k] from Z[k] and Z[M-k] (table
// entries t_k, k <= M/2 only: t_{M-k} = (-t_k.x, t_k.y))
template <typename TT>
struct HilbertMidKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    using Params = HilbertPassParams<T>;
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t row = p.div.div((uint32_t)i), k = (uint32_t)i - row * p.div.d, M = p.len;
        cx<T>* z = p.w + (size_t)row * M;
        if (k == 0) {
            z[0] = mk<T>(0, 0);
            return;
        }
        const cx<T> zk = z[k], zm = z[M - k], tk = ldg(p.tab + k), tm = mk<T>(-tk.x, tk.y);  // t_{M-k}: c -> -c, s -> s
        z[k] = mk<T>(tk.x * zm.x - tk.y * zk.y, tk.y * zk.x - tk.x * zm.y);
        z[M - k] = mk<T>(tm.x * zk.x - tm.y * zm.y, tm.y * zm.x - tm.x * zk.y);
    }
};

// out[2m] = (x[2m], Re w[m]), out[2m+1] = (x[2m+1], Im w[m]): thread i = row M + m (rows are contiguous on both sides)
template <typename TT>
struct HilbertPostKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    using Params = HilbertPassParams<T>;
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const cx<T> xp = ld_stream(reinterpret_cast<const cx<T>*>(p.x) + i), y = p.w[i];
        st_stream(p.out + 2 * i, mk<T>(xp.x, y.x));
        st_stream(p.out + 2 * i + 1, mk<T>(xp.y, y.y));
    }
};

// odd N: out[i] = (x[i], 0)
template <typename TT>
struct HilbertPromoteKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    using Params = HilbertPassParams<T>;
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        p.w[i] = mk<T>(ld_stream_r(p.x + i), (T)0);
    }
};

// odd N: bin k of every row times sgn(k) / N
template <typename TT>
struct HilbertSignKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    using Params = HilbertPassParams<T>;
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t k = (uint32_t)i - p.div.div((uint32_t)i) * p.div.d;
        const T s = k == 0 ? (T)0 : (2 * k < p.len ? p.inv_n : -p.inv_n);
        const cx<T> v = p.w[i];
        p.w[i] = mk<T>(v.x * s, v.y * s);
    }
};

// odd N: the real parts of the output become x
template <typename TT>
struct HilbertRealKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    using Params = HilbertPassParams<T>;
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        st_stream_r(reinterpret_cast<T*>(p.w + i), ld_stream_r(p.x + i));
    }
};

}  // namespace b2
