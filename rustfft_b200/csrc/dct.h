// Real-to-real transforms: DCT-II, DCT-III, DCT-IV and the DSTs of the same types (the `rustdct` layer above RustFFT's Fft
// trait).  Unnormalised; for a row x of length N, n and k in 0 .. N-1:
//     DCT-II   X[k] = sum x[n] cos(pi (2n+1) k / 2N)                                   = scipy.fft.dct(x, 2) / 2
//     DCT-III  X[k] = x[0]/2 + sum_{n>=1} x[n] cos(pi n (2k+1) / 2N)                   = scipy.fft.dct(x, 3) / 2
//     DCT-IV   X[k] = sum x[n] cos(pi (2n+1)(2k+1) / 4N)                               = scipy.fft.dct(x, 4) / 2
// and the DSTs through the same machinery, as index and sign maps on the load and the store:
//     DST-II(x)[k]  = DCT-II((-1)^n x)[N-1-k]      DST-III(x)[k] = (-1)^k DCT-III(x reversed)[k]
//     DST-IV(x)[k]  = (-1)^k DCT-IV(x reversed)[k]
//
// DctKernel<G, KIND>: the whole transform of N = 2M points (M = G::L, a power of two) in one CTA pass, F rows per CTA.
//   load:     the CTA's F rows, contiguous, into shared memory (read as M complex values per row)
//   build:    each thread forms its engine inputs z[m] from shared memory:
//               DCT-II   z[m] = v[2m] + i v[2m+1],  v[j] = x[2j], v[N-1-j] = x[2j+1]                     (Makhoul)
//               DCT-III  V[k] = W_4N^-k (X[k] - i X[N-k]) (X[N] = 0), packed as real.h's inverse packs, times 1/2, then
//                        conjugated: the inverse FFT is conj(FFT(conj .)); the twiddle, pack and 1/2 fold into two table
//                        entries per k (C_k, D_k), rounded once from long double
//               DCT-IV   z[m] = (x[2m] + i x[N-1-2m]) W_8N^(4m+1)
//   engine:   the M-point FFT
//   combine:  DCT-II   Z to shared memory; the pair (k, M-k) gives V[k] = E[k] + W_N^k O[k] (real.h's unpack) and
//                      W_4N^k V[k] = X[k] - i X[N-k] (X[M] = cos(pi/4) (Re Z[0] - Im Z[0]) in place of X[N]), folded into
//                      two table entries per k: W_4N^k V[k] = A_k Z[k] + B_k conj Z[M-k]
//             DCT-III  conjugate, x[2j] = v[j], x[2j+1] = v[N-1-j]
//             DCT-IV   Z[k] W_2N^k = X[2k] - i X[N-1-2k]
//             into shared memory in natural order, then one contiguous store.
// One read and one write of the data and no workspace; every CTA reads its whole rows before it stores, so in place is safe.
// The DST maps are compile-time flags of the kernel: a reversal turns a row offset into a negative one, a sign is a parity known
// at compile time, so no index needs more than a per-thread base and a constant.
//
// DctHalfKernel<T, BASE, 0 | 1>: the pre / post kernels of the general path for even N around the M-point complex plan, one thread
// per k < M and the same algebra and tables as DctKernel (DCT-III: the inverse plan instead of the conjugated forward FFT):
//   DCT-II   pre: z[k] = v[2k] + i v[2k+1];      post: X[k] - i X[N-k] = A_k Z[k] + B_k conj Z[M-k]  (k = 0: X[0], X[M])
//   DCT-III  pre: z[k] = C_k (X[k] - i X[N-k]) + D_k (X[M-k] + i X[M+k]);    post: x[2j] = v[j], x[2j+1] = v[N-1-j]
//   DCT-IV   pre: z[k] = (x[2k] + i x[N-1-2k]) W_8N^(4k+1);                   post: Z[k] W_2N^k = X[2k] - i X[N-1-2k]
// DctGenKernel<T, BASE, 0 | 1>: the pre / post kernels of the general path for odd N around a complex plan, one thread per element:
//   DCT-II   pre: w[n] = v[n] (promoted);                 N-point FFT;   post: X[k] = Re(W_4N^k W[k])
//   DCT-III  pre: w[k] = W_4N^-k (X[k] - i X[N-k]) / 2;    N-point inverse FFT;   post: x[2j] = Re w[j], x[2j+1] = Re w[N-1-j]
//   DCT-IV   pre: w[n] = x[n] W_4N^n, zero for n >= N;     2N-point FFT;  post: X[k] = Re(W_8N^(2k+1) W[k])
#pragma once
#include "kernels.h"

namespace b2 {

enum { DCT_II = 0, DCT_III = 1, DCT_IV = 2 };

template <class G, int KIND>  // KIND: B200FFT_DCT2 .. B200FFT_DST4
struct DctKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int BASE = KIND % 3;  // DCT_II / DCT_III / DCT_IV
    // the DST maps: read x reversed / negate its odd samples, store X reversed / negate its odd outputs
    static constexpr bool IN_REV = KIND == 4 || KIND == 5, IN_ALT = KIND == 3, OUT_REV = KIND == 3, OUT_ALT = KIND == 4 || KIND == 5;
    static constexpr int M = G::L, N = 2 * G::L;
    static constexpr int NT = G::NT;
    // 128 registers per thread where the CTA size allows it (512 threads per SM): the build and combine phases hold the
    // engine's registers plus their twiddles
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, 32);
    static constexpr int P_ENG = 2;                         // phase 0: load, 1: build, then the engine
    static constexpr int P_LAST = P_ENG + Eng::NPHASE - 1;  // last engine phase (its outputs go to shared memory)
    static constexpr int NPHASE = P_LAST + (BASE == DCT_II ? 4 : 2);
    // the F rows, unpadded (row f at reals [f N, (f + 1) N)), in the buffer the engine pads for its own stages
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::F * G::LP;
    static_assert((M & (M - 1)) == 0 && M >= 2, "M must be a power of two");
    static_assert(G::LP >= M, "the rows must fit the engine's buffer");
    struct Params {
        const T* in;
        T* out;
        // k < M:  DCT-II  A_k = W_4N^k (1 - i W_N^k) / 2,       B_k = W_4N^k (1 + i W_N^k) / 2
        //         DCT-III C_k = W_4N^-k (1 + i W_N^-k) / 2,     D_k = W_4N^(M-k) (1 - i W_N^-k) / 2
        //         DCT-IV  W_8N^(4k+1),                         W_2N^k
        const cx<T>* ta;
        const cx<T>* tb;
        const cx<T>* tw;  // stage twiddles of the M-point FFT
        uint64_t rows;    // rows in this launch
        T c8;             // cos(pi/4)
    };
    struct Regs { cx<T> v[G::E]; };

    // input sample n / output k of a row in shared memory, through the kind's maps.  Every index below is a per-thread base plus a
    // compile-time offset (k = j + TP q), and its parity is known at compile time: one address register per row and direction.
    static B2_HD T ld(const T* row, int n) {
        const T v = row[IN_REV ? N - 1 - n : n];
        return (IN_ALT && (n & 1)) ? -v : v;
    }
    static B2_HD void st(T* row, int k, T v) { row[OUT_REV ? N - 1 - k : k] = (OUT_ALT && (k & 1)) ? -v : v; }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        const uint64_t g0 = (uint64_t)bid * G::F;
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        T* row = reinterpret_cast<T*>(smem) + f * N;
        if constexpr (P == 0) {
            // (a whole CTA of rows loads without per-element tests: a row test computed here would be kept live, across every
            // phase, for the store phase's identical test)
            const cx<T>* src = reinterpret_cast<const cx<T>*>(p.in) + g0 * M;
            if (g0 + G::F <= p.rows) {
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) smem[tid + NT * q] = ld_stream(src + tid + NT * q);
            } else {
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const int i = tid + NT * q;
                    smem[i] = g0 + (unsigned)i / M < p.rows ? ld_stream(src + i) : mk<T>(0, 0);
                }
            }
        }
        if constexpr (P == 1) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;  // (k < M/2 exactly when q < E/2)
                if constexpr (BASE == DCT_II) {
                    r.v[q] = q < G::E / 2 ? mk<T>(ld(row, 4 * k), ld(row, 4 * k + 2)) : mk<T>(ld(row, 2 * N - 4 * k - 1), ld(row, 2 * N - 4 * k - 3));
                } else if constexpr (BASE == DCT_III) {
                    // z[k] = C_k (X[k] - i X[N-k]) + D_k (X[M-k] + i X[M+k]), conjugated for the inverse FFT
                    const bool k0 = q == 0 && j == 0;
                    const cx<T> z = cmul(mk<T>(ld(row, k), k0 ? (T)0 : -ld(row, N - k)), ldg(p.ta + k)) +
                                    cmul(mk<T>(ld(row, M - k), ld(row, M + k)), ldg(p.tb + k));
                    r.v[q] = conj(z);
                } else {
                    r.v[q] = cmul(mk<T>(ld(row, 2 * k), ld(row, N - 1 - 2 * k)), ldg(p.ta + k));
                }
            }
        }
        if constexpr (P >= P_ENG && P <= P_LAST) Eng::template phase<P - P_ENG>(tid, r.v, smem, p.tw);
        if constexpr (P == P_LAST) {
            // the engine's last phase reads no shared memory: the rows can be overwritten now
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                if constexpr (BASE == DCT_II) {
                    smem[f * M + k] = r.v[q];
                } else if constexpr (BASE == DCT_III) {
                    const cx<T> c = conj(r.v[q]);  // v[2k] + i v[2k+1]
                    if (q < G::E / 2) {
                        st(row, 4 * k, c.x);
                        st(row, 4 * k + 2, c.y);
                    } else {
                        st(row, 2 * N - 4 * k - 1, c.x);
                        st(row, 2 * N - 4 * k - 3, c.y);
                    }
                } else {
                    const cx<T> y = cmul(r.v[q], ldg(p.tb + k));
                    st(row, 2 * k, y.x);
                    st(row, N - 1 - 2 * k, -y.y);
                }
            }
        }
        if constexpr (BASE == DCT_II && P == P_LAST + 1) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                const bool k0 = q == 0 && j == 0;
                const cx<T> zk = r.v[q], zm = conj(smem[f * M + (k0 ? 0 : M - k)]);
                // W_4N^k V[k] = A_k Z[k] + B_k conj Z[M-k] = X[k] - i X[N-k];  k = 0: X[M] = cos(pi/4) (Re Z[0] - Im Z[0])
                const cx<T> u = cmul(zk, ldg(p.ta + k)) + cmul(zm, ldg(p.tb + k));
                r.v[q] = mk<T>(u.x, k0 ? p.c8 * (zk.x - zk.y) : -u.y);
            }
        }
        if constexpr (BASE == DCT_II && P == P_LAST + 2) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                st(row, k, r.v[q].x);
                if (q == 0 && j == 0) st(row, M, r.v[q].y);
                else st(row, N - k, r.v[q].y);
            }
        }
        if constexpr (P == NPHASE - 1) {
            cx<T>* dst = reinterpret_cast<cx<T>*>(p.out) + g0 * M;
            if (g0 + G::F <= p.rows) {
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) st_stream(dst + tid + NT * q, smem[tid + NT * q]);
            } else {
                const unsigned last = (unsigned)(p.rows - g0) * M;  // elements of the rows that exist
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const unsigned i = tid + NT * q;
                    if (i < last) st_stream(dst + i, smem[i]);
                }
            }
        }
    }
};

// general path, even N: one thread per k < M of a row (pre: M workspace values, post: two outputs)
template <typename TT, int BASE, int DIR>  // DIR 0: pre (signal -> complex workspace), 1: post (workspace -> result)
struct DctHalfKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const void* in;
        void* out;
        const cx<T>* ta;  // the DctKernel tables of N: M entries each
        const cx<T>* tb;
        uint64_t n_elem;  // rows * M
        uint32_t N;
        FastDiv div_m;    // by M
        T c8;             // cos(pi/4)
        bool in_rev, out_rev, in_alt, out_alt;
    };
    struct Regs {};
    static B2_HD T ld(const Params& p, const T* x, uint32_t n) {
        const T v = x[p.in_rev ? p.N - 1 - n : n];
        return (p.in_alt && (n & 1)) ? -v : v;
    }
    static B2_HD void st(const Params& p, T* x, uint32_t k, T v) { x[p.out_rev ? p.N - 1 - k : k] = (p.out_alt && (k & 1)) ? -v : v; }
    // Makhoul's permutation: v[n] = x[2n] (n < M), x[2N - 2n - 1] (n >= M)
    static B2_HD uint32_t perm(uint32_t n, uint32_t N) { return 2 * n < N ? 2 * n : 2 * N - 2 * n - 1; }
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t M = p.div_m.d, N = p.N, row = p.div_m.div((uint32_t)i), k = (uint32_t)i - row * M;
        if (DIR == 0) {
            const T* x = (const T*)p.in + (uint64_t)row * N;
            cx<T> z;
            if (BASE == DCT_II) {
                z = mk<T>(ld(p, x, perm(2 * k, N)), ld(p, x, perm(2 * k + 1, N)));
            } else if (BASE == DCT_III) {
                z = cmul(mk<T>(ld(p, x, k), k ? -ld(p, x, N - k) : (T)0), ldg(p.ta + k)) +
                    cmul(mk<T>(ld(p, x, M - k), ld(p, x, M + k)), ldg(p.tb + k));
            } else {
                z = cmul(mk<T>(ld(p, x, 2 * k), ld(p, x, N - 1 - 2 * k)), ldg(p.ta + k));
            }
            ((cx<T>*)p.out)[i] = z;
        } else {
            const cx<T>* z = (const cx<T>*)p.in + (uint64_t)row * M;
            T* x = (T*)p.out + (uint64_t)row * N;
            if (BASE == DCT_II) {
                const cx<T> zk = z[k], zm = conj(z[k ? M - k : 0]);
                const cx<T> u = cmul(zk, ldg(p.ta + k)) + cmul(zm, ldg(p.tb + k));
                st(p, x, k, u.x);
                if (k) st(p, x, N - k, -u.y);
                else st(p, x, M, p.c8 * (zk.x - zk.y));
            } else if (BASE == DCT_III) {
                const cx<T> c = z[k];  // v[2k] + i v[2k+1]
                st(p, x, perm(2 * k, N), c.x);
                st(p, x, perm(2 * k + 1, N), c.y);
            } else {
                const cx<T> y = cmul(z[k], ldg(p.tb + k));
                st(p, x, 2 * k, y.x);
                st(p, x, N - 1 - 2 * k, -y.y);
            }
        }
    }
};

// general path, odd N: one element per thread; rows of `len` outputs (pre: the workspace, post: the result)
template <typename TT, int BASE, int DIR>  // DIR 0: pre (signal -> complex workspace), 1: post (workspace -> result)
struct DctGenKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const void* in;
        void* out;
        const cx<T>* ta;  // DCT-II / III: W_4N^k, k < N;   DCT-IV: W_4N^n, n < N
        const cx<T>* tb;  // DCT-IV: W_8N^(2k+1), k < N
        uint64_t n_elem;  // rows * len
        uint32_t N, wlen;  // transform length, workspace row length (N, or 2N for DCT-IV)
        FastDiv div_len;   // by the row length this launch walks (pre: wlen, post: N)
        bool in_rev, out_rev, in_alt, out_alt;
    };
    struct Regs {};
    static B2_HD T ld(const Params& p, const T* x, uint32_t n) {
        const T v = x[p.in_rev ? p.N - 1 - n : n];
        return (p.in_alt && (n & 1)) ? -v : v;
    }
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t len = p.div_len.d, row = p.div_len.div((uint32_t)i), e = (uint32_t)i - row * len, N = p.N;
        if (DIR == 0) {
            const T* x = (const T*)p.in + (uint64_t)row * N;
            cx<T> w;
            if (BASE == DCT_II) {
                w = mk<T>(ld(p, x, 2 * e < N ? 2 * e : 2 * N - 2 * e - 1), (T)0);
            } else if (BASE == DCT_III) {
                const cx<T> v = cmulc(mk<T>(ld(p, x, e), e ? -ld(p, x, N - e) : (T)0), ldg(p.ta + e));
                w = mk<T>(v.x * (T)0.5, v.y * (T)0.5);
            } else {
                w = e < N ? cmul(mk<T>(ld(p, x, e), (T)0), ldg(p.ta + e)) : mk<T>(0, 0);
            }
            ((cx<T>*)p.out)[i] = w;
        } else {
            const cx<T>* w = (const cx<T>*)p.in + (uint64_t)row * p.wlen;
            T v;
            if (BASE == DCT_II) v = cmul(w[e], ldg(p.ta + e)).x;
            else if (BASE == DCT_III) v = w[(e & 1) ? N - (e + 1) / 2 : e / 2].x;
            else v = cmul(w[e], ldg(p.tb + e)).x;
            ((T*)p.out)[(uint64_t)row * N + (p.out_rev ? N - 1 - e : e)] = (p.out_alt && (e & 1)) ? -v : v;
        }
    }
};

// DctAxisKernel<G, KIND>: DctKernel<G, KIND> down a strided axis, for the 2-D / 3-D transforms.  The data is viewed as
// [outer][N][inner] (N = 2M, M = G::L); column g = o inner + c (o < outer, c < inner) holds element n at o N inner + n inner + c.  A CTA
// takes the F adjacent columns g0 .. g0 + F - 1 (a tile may span slabs, and in a launch's last CTA it may end early):
//   phase 0      the [N][F] tile from global memory, a warp reading runs of F adjacent columns per row (coalesced), into registers,
//                then into a staging layout of the same buffer: element (n, f) at real n F + ((f + rot(n)) mod F)
//   phase 1      the staging layout into registers: thread t's slot k is real t + NT k of the layout below or, where a column
//                spans at least a 128-byte run of threads (BY_COLUMN), row t mod RS + RS k of column t / RS (RS = NT / F)
//   phase 2      registers into DctKernel's layout: column f at reals [f N, (f + 1) N)
//   then DctKernel's phases 1 .. NPHASE - 2 (build, M-point engine, combine) unchanged, on an embedded DctKernel::Params,
//   and the reverse: DctKernel's layout -> registers -> staging -> registers -> global memory.
// rot(n) = n max(1, B/N) / max(1, B/F), B = reals per 128 bytes: a warp's accesses of the staging in either order fall on distinct
// banks, and DctKernel's layout is accessed at consecutive reals (tests/test_dctn.py enumerates every warp access of both).  In the
// column order every address of a thread is one base plus compile-time offsets; the order of DctKernel's layout made f32 M >= 256
// spill (each slot's staging address computed separately).  Every CTA reads its whole tile before it stores, so in place is safe;
// no workspace.
template <class G, int KIND>
struct DctAxisKernel {
    using T = typename G::T;
    using DK = DctKernel<G, KIND>;
    static constexpr int M = G::L, N = 2 * G::L, F = G::F, NT = G::NT;
    static constexpr int K = N * F / NT;  // reals per thread in the load and the store (2 E: DctKernel's registers)
    static constexpr int RS = NT / F;     // rows of the tile one load / store slot covers
    static constexpr int B = 128 / (int)sizeof(T);
    static constexpr int ROT_MUL = N < B ? B / N : 1, ROT_DIV = F < B ? B / F : 1;
    // column order in phases 1 / 2 and their reverse: a warp's run of B threads stays in one column, and row n + RS k of a column is
    // staged RS F k reals after row n (RS / ROT_DIV, the rotation's step, is a multiple of F)
    static constexpr bool BY_COLUMN = RS >= B && (RS / ROT_DIV) % F == 0;
    // the same step for the rows of the load and the store: row n0 + RS k of a column staged RS F k reals after row n0
    static constexpr bool ROW_STEP = (RS * ROT_MUL) % ROT_DIV == 0 && (RS * ROT_MUL / ROT_DIV) % F == 0;
    static constexpr int MIN_BLOCKS = DK::MIN_BLOCKS;
    static constexpr int P_DK = 2;                       // DctKernel's phase P (1 .. DK::NPHASE - 2) runs as phase P + P_DK
    static constexpr int P_OUT = DK::NPHASE - 1 + P_DK;  // first phase of the store
    static constexpr int NPHASE = P_OUT + 3;
    static constexpr size_t SMEM_BYTES = DK::SMEM_BYTES;
    static_assert(K == 2 * G::E && NT % F == 0 && (F & (F - 1)) == 0, "the tile must split evenly over the threads");
    static_assert((size_t)N * F * sizeof(T) <= SMEM_BYTES, "the tile must fit DctKernel's buffer");
    struct Params {
        typename DK::Params dk;  // DctKernel's tables (its in / out / rows are not used)
        const T* in;
        T* out;
        uint64_t cols;       // columns in this launch (cols + F < 2^31)
        uint64_t slab;       // elements between slabs: N inner
        uint64_t row;        // elements between the rows of a column: inner
        FastDiv div_inner;   // g -> (o, c); a launch inside one slab divides by 2^30 (o = 0)
    };
    using Regs = typename DK::Regs;

    static B2_HD int stage(int n, int f) { return n * F + ((f + n * ROT_MUL / ROT_DIV) & (F - 1)); }
    static B2_HD T& reg(Regs& r, int k) { return (k & 1) ? r.v[k >> 1].y : r.v[k >> 1].x; }
    // staging real of the load's / store's slot k (row tid / F + RS k of column tid mod F)
    static B2_HD int row_slot(int tid, int k) {
        if constexpr (ROW_STEP) return stage(tid / F, tid & (F - 1)) + RS * F * k;
        else return stage(tid / F + RS * k, tid & (F - 1));
    }
    // slot k of thread tid in phases 1 / 2 and their reverse: its real in DctKernel's layout and in the staging layout
    static B2_HD void slot(int tid, int k, int& fin, int& stg) {
        if constexpr (BY_COLUMN) {
            const int f = tid / RS, j = tid % RS;
            fin = f * N + j + RS * k;
            stg = stage(j, f) + RS * F * k;
        } else {
            const int i = tid + NT * k;
            fin = i;
            stg = stage(i % N, i / N);
        }
    }
    // offset of row tid / F of this thread's column g0 + tid mod F
    static B2_HD uint64_t origin(const Params& p, uint32_t bid, int tid) {
        const uint32_t g = bid * F + (tid & (F - 1)), o = p.div_inner.div(g);
        return (uint64_t)o * p.slab + (g - o * p.div_inner.d) + (uint64_t)(tid / F) * p.row;
    }
    static B2_HD bool whole(const Params& p, uint32_t bid) { return (uint64_t)bid * F + F <= p.cols; }
    static B2_HD bool live(const Params& p, uint32_t bid, int tid) { return (uint64_t)bid * F + (tid & (F - 1)) < p.cols; }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        T* s = reinterpret_cast<T*>(smem);
        if constexpr (P == 0) {
            // (only a launch's last CTA tests its columns; one test per thread: a thread keeps one column)
            if (whole(p, bid) || live(p, bid, tid)) {
                const T* src = p.in + origin(p, bid, tid);
                const uint64_t step = (uint64_t)RS * p.row;
                B2_UNROLL
                for (int k = 0; k < K; ++k) reg(r, k) = src[k * step];
            } else {
                B2_UNROLL
                for (int k = 0; k < K; ++k) reg(r, k) = (T)0;
            }
            B2_UNROLL
            for (int k = 0; k < K; ++k) s[row_slot(tid, k)] = reg(r, k);
        }
        if constexpr (P == 1 || P == 2 || P == P_OUT || P == P_OUT + 1) {
            B2_UNROLL
            for (int k = 0; k < K; ++k) {
                int fin, stg;
                slot(tid, k, fin, stg);
                if constexpr (P == 1) reg(r, k) = s[stg];
                if constexpr (P == 2) s[fin] = reg(r, k);
                if constexpr (P == P_OUT) reg(r, k) = s[fin];
                if constexpr (P == P_OUT + 1) s[stg] = reg(r, k);
            }
        }
        if constexpr (P > P_DK && P < P_OUT) DK::template phase<P - P_DK>(p.dk, bid, tid, r, smem);
        if constexpr (P == P_OUT + 2) {
            B2_UNROLL
            for (int k = 0; k < K; ++k) reg(r, k) = s[row_slot(tid, k)];
            if (whole(p, bid) || live(p, bid, tid)) {
                T* dst = p.out + origin(p, bid, tid);
                const uint64_t step = (uint64_t)RS * p.row;
                B2_UNROLL
                for (int k = 0; k < K; ++k) dst[k * step] = reg(r, k);
            }
        }
    }
};

// DctTransposeKernel<T>: out[s os + c ol + r] = in[s is + r il + c] for r < R, c < C, s < slabs: the transposition of each [R][C] slab
// around the 1-D plan on the N-D transforms' other route.  32 x 32 tiles through shared memory padded to a pitch of 33, 256 threads;
// reads along c and writes along r are coalesced, and both shared-memory sides are free of bank conflicts (tests/test_dctn.py).
template <typename TT>
struct DctTransposeKernel {
    using T = TT;
    static constexpr int TILE = 32, PITCH = TILE + 1;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 2;
    static constexpr size_t SMEM_BYTES = sizeof(T) * TILE * PITCH;
    struct Params {
        const T* in;
        T* out;
        uint32_t R, C;     // rows and columns of a slab
        uint32_t tr, tc;   // tiles along R and C
        uint64_t is, il;   // input: elements between slabs, between rows
        uint64_t os, ol;   // output: elements between slabs, between columns
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>* smem) {
        T* tile = reinterpret_cast<T*>(smem);
        const uint32_t bc = bid % p.tc, t = bid / p.tc, br = t % p.tr, sl = t / p.tr;
        const int x = tid % TILE, y = tid / TILE;
        if constexpr (P == 0) {
            const uint32_t c = bc * TILE + x;
            const T* src = p.in + sl * p.is + c;
            B2_UNROLL
            for (int i = 0; i < TILE; i += NT / TILE) {
                const uint32_t r = br * TILE + y + i;
                if (r < p.R && c < p.C) tile[(y + i) * PITCH + x] = src[r * p.il];
            }
        } else {
            const uint32_t r = br * TILE + x;
            T* dst = p.out + sl * p.os + r;
            B2_UNROLL
            for (int i = 0; i < TILE; i += NT / TILE) {
                const uint32_t c = bc * TILE + y + i;
                if (r < p.R && c < p.C) dst[c * p.ol] = tile[x * PITCH + y + i];
            }
        }
    }
};

}  // namespace b2
