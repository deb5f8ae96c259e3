// Kernel bodies (phase functions) built on the CTA engine, and the global-memory functors that
// give each its role:
//
//   FftKernel<G, M0, M1, Load, Store>   one FFT pass: Load -> L-point FFT -> Store
//       Load = LoadRows,  Store = StoreRows            whole transform in one CTA pass  (N = L)
//       Load = LoadCols,  Store = StoreCols            four-step pass A: strided column FFTs of
//                                                      length N1, in place
//       Load = LoadRowsTw, Store = StoreTransposed     four-step pass B: contiguous rows times
//                                                      W_N^(n2*k1), N2-point FFT, written transposed
//   (four-step == the reference's six-step MixedRadix, src/algorithm/mixed_radix.rs:128-158, with
//    its three transposes folded into the strided loads/stores of the two passes)
//
//   BluesteinKernel<G>   whole chirp-z transform of one signal in one CTA pass
//                        (src/algorithm/bluesteins_algorithm.rs:100-136 fused: x*w -> FFT_M ->
//                         *C, conj -> FFT_M -> conj * w; with separate input / output lengths and
//                         tables it is the CZT of any arc on the unit circle)
//   RaderKernel<G>       whole Rader transform of one prime-length signal in one CTA pass
//                        (src/algorithm/raders_algorithm.rs:235-283 fused)
//
// Direction: every table is "forward".  An inverse plan sets SWAP on the outermost load and the
// outermost store (ifft(x) = swap(fft(swap(x))), swap = exchange re/im) -- see common.h.
#pragma once
#include "engine.h"
#include "tma.h"

namespace b2 {

// resident CTAs per SM the register allocator must leave room for: 64 registers per thread for the
// 16-element geometries (2048 threads per SM), 128 for the 32-element (radix-32) ones
constexpr int default_min_blocks(int nt, int e = 16) {
    const int target_threads = e >= 24 ? 512 : 1024;
    const int b = target_threads / nt;
    return b < 1 ? 1 : (b > 8 ? 8 : b);
}

// unsigned division by a run-time constant through a precomputed reciprocal (the stage geometry of the
// SmoothKernel is run-time data; plain `/` and `%` cost ~20 instructions each)
struct FastDiv {
    uint32_t d, mul, shift;  // q = umulhi(n, mul) >> shift   (n < 2^31)
    B2_HD uint32_t div(uint32_t n) const {
        if (d == 1) return n;
#if defined(__CUDA_ARCH__)
        return __umulhi(n, mul) >> shift;
#else
        return (uint32_t)(((uint64_t)n * mul) >> 32) >> shift;
#endif
    }
};
inline FastDiv make_fastdiv(uint32_t d) {
    FastDiv f{d, 0, 0};
    if (d <= 1) return f;
    uint32_t l = 0;
    while ((1u << l) < d) ++l;  // ceil(log2 d)
    // round-up method, exact for n < 2^31
    const uint64_t m = ((1ull << (32 + l)) + d - 1) / d;
    if (m < (1ull << 32)) {
        f.mul = (uint32_t)m;
        f.shift = l;
    } else {  // m needs 33 bits: use l-1 (still exact for n < 2^31 because d > 2^(l-1))
        f.mul = (uint32_t)(((1ull << (32 + l - 1)) + d - 1) / d);
        f.shift = l - 1;
    }
    return f;
}

// ------------------------------------------------------------------------------------------
// Functors.  prep(g, ok) is evaluated once per thread (g = global FFT index of this thread's
// FFT, ok = g is inside the launch), get/put once per element.
// ------------------------------------------------------------------------------------------
template <typename T, bool SWAP>
struct LoadRows {  // element e of FFT g at in[g*len + e]
    const cx<T>* in;
    uint32_t len;
    struct St { const cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const { return St{in + g * (uint64_t)len, ok}; }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        cx<T> v = ld_stream(s.p + e);
        return SWAP ? swap_ri(v) : v;
    }
};

template <typename T, bool SWAP>
struct StoreRows {
    cx<T>* out;
    uint32_t len;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const { return St{out + g * (uint64_t)len, ok}; }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) st_stream(s.p + e, SWAP ? swap_ri(v) : v);
    }
};

// four-step pass A load: FFT g = (transform b, column c) with g = b*N2 + c; element e (= n1) lives
// at in[b*N + e*N2 + c].  N2 = 1 << lg2.
template <typename T, bool SWAP>
struct LoadCols {
    const cx<T>* in;
    uint32_t lgN;   // log2 N
    uint32_t lg2;   // log2 N2
    struct St { const cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = g >> lg2, c = g & ((1ull << lg2) - 1);
        return St{in + (b << lgN) + c, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        cx<T> v = ld_cs(s.p + ((uint32_t)e << lg2));
        return SWAP ? swap_ri(v) : v;
    }
};

// four-step pass A store: out[b*N + k1*N2 + c] = v  (the slots the tile was read from, so the pass is in
// place per tile; plain write-back stores: pass B re-reads them from L2)
template <typename T>
struct StoreCols {
    cx<T>* out;
    uint32_t lgN, lg2;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = g >> lg2, c = g & ((1ull << lg2) - 1);
        return St{out + (b << lgN) + c, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) s.p[(uint32_t)e << lg2] = v;  // plain write-back store: pass B re-reads it from L2
    }
};

// four-step pass B load: row k1 of transform b (FFT g = b*N1 + k1), element n2 = e, times the inter-pass
// twiddle W_N^(k1*n2) from a full [k1][n2] table (N entries, each rounded once from long double --
// the reference's MixedRadix keeps the same N-entry table, src/algorithm/mixed_radix.rs:66-71).
// The table is applied HERE rather than on pass A's store because this side is contiguous: table and
// data are both read as 256-byte-per-warp streams (round 1 measured the earlier two-level gather on the
// strided side as the LSU-pipe bottleneck of pass A).
template <typename T>
struct LoadRowsTw {
    const cx<T>* in;
    const cx<T>* tw;  // [N1][N2]
    uint32_t len;     // N2
    uint32_t lg1;     // log2 N1
    uint32_t discard = 0;  // 1: `in` is dead scratch once read -- drop its lines from L2 without write-back
    // called by every thread once ALL threads of the CTA hold their inputs in registers: the F rows of a tile are
    // one contiguous, 128-byte aligned block of F*len elements starting at FFT g0
    B2_HD void tile_done(uint64_t g0, uint32_t n_ffts, int tid, int nt) const {
        if (!discard) return;
        const char* base = reinterpret_cast<const char*>(in + g0 * (uint64_t)len);
        const uint32_t lines = (uint32_t)((uint64_t)n_ffts * len * sizeof(cx<T>) / 128);
        for (uint32_t l = (uint32_t)tid; l < lines; l += (uint32_t)nt) l2_discard_line(base + (size_t)l * 128);
    }
    static constexpr bool HAS_TILE_DONE = true;
    struct St { const cx<T>* p; const cx<T>* t; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t k1 = g & ((1ull << lg1) - 1);
        return St{in + g * (uint64_t)len, tw + k1 * (uint64_t)len, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        return cmul(ld_cs(s.p + e), ldg_stream(s.t + e));
    }
};

// four-step pass B store: FFT g = (transform b, row k1), g = b*N1 + k1; output k2 (= e) goes to
// out[b*N + k1 + N1*e].  N1 = 1 << lg1.
template <typename T, bool SWAP>
struct StoreTransposed {
    cx<T>* out;
    uint32_t lgN, lg1;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = g >> lg1, k1 = g & ((1ull << lg1) - 1);
        return St{out + (b << lgN) + k1, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) st_cs(s.p + ((uint32_t)e << lg1), SWAP ? swap_ri(v) : v);
    }
};

// ---- the same four functors for ARBITRARY N1, N2 (compiled two-pass plans of composite lengths: 10000 = 100 x 100,
// 44100 = 196 x 225, 48000 = 128 x 375, 10^6 = 1000 x 1000): shifts become multiplications, g -> (transform, column | row)
// goes through a precomputed reciprocal.  The reference's MixedRadix for the same sizes: src/algorithm/mixed_radix.rs:128-158.
template <typename T, bool SWAP>
struct LoadColsG {  // pass A: FFT g = (b, c), g = b*N2 + c; element e at in[b*N + e*N2 + c]
    const cx<T>* in;
    uint64_t N;
    uint32_t N2;
    FastDiv div2;
    struct St { const cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t b = div2.div((uint32_t)g), c = (uint32_t)g - b * N2;
        return St{in + (uint64_t)b * N + c, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        cx<T> v = ld_cs(s.p + (size_t)e * N2);
        return SWAP ? swap_ri(v) : v;
    }
};
template <typename T>
struct StoreColsG {  // pass A: out[b*N + k1*N2 + c] (the slots the tile was read from)
    cx<T>* out;
    uint64_t N;
    uint32_t N2;
    FastDiv div2;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t b = div2.div((uint32_t)g), c = (uint32_t)g - b * N2;
        return St{out + (uint64_t)b * N + c, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) s.p[(size_t)e * N2] = v;  // plain write-back store: pass B re-reads it from L2
    }
};
template <typename T>
struct LoadRowsTwG {  // pass B: row k1 of transform b (g = b*N1 + k1), element n2 = e, times W_N^(k1 n2) from the [k1][n2] table
    const cx<T>* in;
    const cx<T>* tw;
    uint32_t len;  // N2
    uint32_t N1;
    FastDiv div1;
    uint32_t discard = 0;
    B2_HD void tile_done(uint64_t g0, uint32_t n_ffts, int tid, int nt) const {
        if (!discard) return;
        const uint64_t bytes = (uint64_t)n_ffts * len * sizeof(cx<T>), off = g0 * (uint64_t)len * sizeof(cx<T>);
        if ((bytes | off) & 127u) return;  // whole, aligned 128-byte lines only
        const char* base = reinterpret_cast<const char*>(in) + off;
        for (uint32_t l = (uint32_t)tid; l < (uint32_t)(bytes / 128); l += (uint32_t)nt) l2_discard_line(base + (size_t)l * 128);
    }
    static constexpr bool HAS_TILE_DONE = true;
    struct St { const cx<T>* p; const cx<T>* t; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t b = div1.div((uint32_t)g), k1 = (uint32_t)g - b * N1;
        return St{in + g * (uint64_t)len, tw + (uint64_t)k1 * len, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        return cmul(ld_cs(s.p + e), ldg_stream(s.t + e));
    }
};
template <typename T, bool SWAP>
struct StoreTransposedG {  // pass B: output k2 = e of row k1 goes to out[b*N + k1 + N1*e]
    cx<T>* out;
    uint64_t N;
    uint32_t N1;
    FastDiv div1;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t b = div1.div((uint32_t)g), k1 = (uint32_t)g - b * N1;
        return St{out + (uint64_t)b * N + k1, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) st_cs(s.p + (size_t)e * N1, SWAP ? swap_ri(v) : v);
    }
};

// ---- ring-addressed workspace functors of the single-launch dataflow four-step (run_flow below) ----
// The intermediate of transform b lives in slot (b mod ring_w) of a small ring of N-element slots that
// stays L2 resident; everything else is as in StoreCols / LoadRowsTw.
template <typename T>
struct StoreColsRing {
    cx<T>* out;
    uint32_t lgN, lg2, ring_w;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = (uint32_t)(g >> lg2) % ring_w, c = g & ((1ull << lg2) - 1);
        return St{out + (b << lgN) + c, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) s.p[(uint32_t)e << lg2] = v;  // plain write-back store: pass B re-reads it from L2
    }
};
template <typename T>
struct LoadRowsTwRing {
    const cx<T>* in;
    const cx<T>* tw;  // [N1][N2]
    uint32_t len;     // N2
    uint32_t lg1;     // log2 N1
    uint32_t lgN, ring_w;
    uint32_t discard = 0;  // as in LoadRowsTw
    B2_HD void tile_done(uint64_t g0, uint32_t n_ffts, int tid, int nt) const {
        if (!discard) return;
        const uint64_t k1 = g0 & ((1ull << lg1) - 1), b = (uint32_t)(g0 >> lg1) % ring_w;
        const char* base = reinterpret_cast<const char*>(in + (b << lgN) + k1 * (uint64_t)len);
        const uint32_t lines = (uint32_t)((uint64_t)n_ffts * len * sizeof(cx<T>) / 128);
        for (uint32_t l = (uint32_t)tid; l < lines; l += (uint32_t)nt) l2_discard_line(base + (size_t)l * 128);
    }
    static constexpr bool HAS_TILE_DONE = true;
    struct St { const cx<T>* p; const cx<T>* t; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t k1 = g & ((1ull << lg1) - 1), b = (uint32_t)(g >> lg1) % ring_w;
        return St{in + (b << lgN) + k1 * (uint64_t)len, tw + k1 * (uint64_t)len, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        // strong (L1-bypassing) load: the slot was written by other SMs during this launch
        return cmul(ld_strong(s.p + e), ldg_stream(s.t + e));
    }
#if defined(B2_TWROW_FEW)
    // all E elements of thread j at once: W_N^(k1 (j + TP q)) = W_N^(k1 j) * W_N^(k1 TP q).  Both factors are entries
    // of table row k1 (columns j and TP q); only the columns TP 2^i are loaded (the same address for every thread
    // of a row: a broadcast) and the other powers are built as products -- 1 + log2 E table loads instead of E.
    static constexpr bool HAS_LOAD_ALL = sizeof(T) == 4;
    template <int E, int TP>
    B2_HD void load_all(const St& s, int j, cx<T> (&v)[E]) const {
        B2_UNROLL
        for (int q = 0; q < E; ++q) v[q] = ld_strong(s.p + j + TP * q);
        cx<T> w[E];
        const cx<T> a = ldg_stream(s.t + j);
        B2_UNROLL
        for (int q = 1; q < E; q <<= 1) w[q] = ldg_stream(s.t + TP * q);
        B2_UNROLL
        for (int q = 3; q < E; ++q)
            if (q & (q - 1)) w[q] = cmul(w[hibit(q)], w[q - hibit(q)]);
        v[0] = cmul(v[0], a);
        B2_UNROLL
        for (int q = 1; q < E; ++q) v[q] = cmul(v[q], cmul(a, w[q]));
    }
#else
    static constexpr bool HAS_LOAD_ALL = false;
#endif
};

// ------------------------------------------------------------------------------------------
// Functors of the large convolution plans (Rader / Bluestein with an inner FFT of M = N1*N2 > one
// CTA): the same two four-step passes, with the algorithm's gather / chirp / pointwise / scatter
// steps folded into the first pass' loads and the second pass' stores, so no step of
// src/algorithm/raders_algorithm.rs:235-283 / bluesteins_algorithm.rs:100-136 is a separate sweep
// over memory.
// ------------------------------------------------------------------------------------------
// pass A load of the FIRST inner FFT.  Inner element i = e*N2 + c of transform b comes from
//   gather != null (Rader):     in[b*n + gather[i]]            gather[i] = g^(i+1) mod n
//   gather == null (Bluestein): i < n ? in[b*n + i] * chirp[i] : 0
template <typename T, bool SWAP>
struct LoadColsConv {
    const cx<T>* in;
    const uint32_t* gather;
    const cx<T>* chirp;
    uint32_t n;    // outer length = stride between transforms of `in`
    uint32_t lg2;  // log2 N2 (inner)
    struct St { const cx<T>* p; uint32_t c; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = g >> lg2;
        return St{in + b * (uint64_t)n, (uint32_t)(g & ((1ull << lg2) - 1)), ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        const uint32_t i = ((uint32_t)e << lg2) + s.c;
        if (gather) {
            cx<T> v = s.p[ldg_u32(gather + i)];
            return SWAP ? swap_ri(v) : v;
        }
        if (i >= n) return mk<T>(0, 0);
        cx<T> v = ld_stream(s.p + i);
        if (SWAP) v = swap_ri(v);
        return cmul(v, ldg(chirp + i));
    }
};

// pass B store of the inner FFTs.  FFT g = (transform b, row k1); output e lands on inner index
// k = k1 + N1*e.
//   MODE 0 (end of inner FFT #1): work[b*M + k] = conj(v * mult[k]); Rader (x_in != null) also does
//           the DC bookkeeping at k == 0:  out[b*n] = x0 + v,  and adds conj(x0) to the stored value
//   MODE 1 (end of inner FFT #2, Rader):     out[b*n + scatter[k]] = conj(v)    scatter[k] = g^-(k+1) mod n
//   MODE 2 (end of inner FFT #2, Bluestein): k < n: out[b*n + k] = conj(v) * chirp[k]
template <typename T, bool SWAP, int MODE>
struct StoreTransposedConv {
    cx<T>* out;            // MODE 0: work (stride M); MODE 1/2: user output (stride n)
    const cx<T>* mult;     // MODE 0
    const uint32_t* scatter;  // MODE 1
    const cx<T>* chirp;    // MODE 2
    const cx<T>* x_in;     // MODE 0, Rader: user input (stride n), else null
    cx<T>* x_out;          // MODE 0, Rader: user output (stride n)
    uint32_t n;            // outer length
    uint32_t lgM, lg1;
    struct St { cx<T>* p; uint64_t b; uint32_t k1; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint64_t b = g >> lg1;
        const uint32_t k1 = (uint32_t)(g & ((1ull << lg1) - 1));
        cx<T>* p = (MODE == 0) ? out + (b << lgM) : out + b * (uint64_t)n;
        return St{p, b, k1, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (!s.ok) return;
        const uint32_t k = s.k1 + ((uint32_t)e << lg1);
        if (MODE == 0) {
            cx<T> w = conj(cmul(v, ldg(mult + k)));
            if (x_in != nullptr && k == 0) {
                cx<T> x0 = x_in[s.b * (uint64_t)n];
                if (SWAP) x0 = swap_ri(x0);
                const cx<T> dc = x0 + v;
                x_out[s.b * (uint64_t)n] = SWAP ? swap_ri(dc) : dc;
                w = w + conj(x0);
            }
            s.p[k] = w;
        } else if (MODE == 1) {
            const cx<T> w = conj(v);
            s.p[ldg_u32(scatter + k)] = SWAP ? swap_ri(w) : w;
        } else {
            if (k < n) {
                const cx<T> w = cmul(conj(v), ldg(chirp + k));
                st_stream(s.p + k, SWAP ? swap_ri(w) : w);
            }
        }
    }
};

// ------------------------------------------------------------------------------------------
// a Load functor may provide load_all<E, TP>(st, j, v) (all elements of a thread at once) and say so with HAS_LOAD_ALL
template <class L, class = void> struct load_all_of { static constexpr bool value = false; };
template <class L> struct load_all_of<L, decltype((void)L::HAS_LOAD_ALL)> { static constexpr bool value = L::HAS_LOAD_ALL; };

template <class L, class = void> struct tile_done_of { static constexpr bool value = false; };
template <class L> struct tile_done_of<L, decltype((void)L::HAS_TILE_DONE)> { static constexpr bool value = L::HAS_TILE_DONE; };

template <class G, Map M0, Map M1, class Load, class Store>
struct FftKernel {
    using T = typename G::T;
    using Eng = Engine<G, M0, M1>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, G::E);
    static constexpr int NPHASE = Eng::NPHASE;
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::SMEM_ELEMS;
    struct Params {
        Load load;
        Store store;
        const cx<T>* tw;   // packed stage twiddles, RL::tw_total() entries
        uint64_t n_fft;    // FFTs in this launch
    };
    struct Regs { cx<T> v[G::E]; };

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        if constexpr (P == 0) {
            int f, j;
            Eng::template owner<0>(tid, f, j);
            // FFTs past the end of the launch (last CTA of a ragged batch) re-read the last valid FFT
            // instead of predicating every load; their stores are masked below
            uint64_t g = (uint64_t)bid * G::F + f;
            if (g >= p.n_fft) g = p.n_fft - 1;
            const auto st = p.load.prep(g, true);
            if constexpr (load_all_of<Load>::value) {
                p.load.template load_all<G::E, G::TP>(st, j, r.v);
            } else {
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) r.v[q] = p.load.get(st, j + G::TP * q);
            }
        }
        if constexpr (P == 1 && tile_done_of<Load>::value) {
            // the barrier before this phase: every thread of the CTA has consumed its loads
            const uint64_t g0 = (uint64_t)bid * G::F;
            if (g0 + G::F <= p.n_fft) p.load.tile_done(g0, (uint32_t)G::F, tid, G::NT);
        }
        Eng::template phase<P>(tid, r.v, smem, p.tw);
        if constexpr (P == NPHASE - 1) {
            int f, j;
            Eng::out_owner(tid, f, j);
            const uint64_t g = (uint64_t)bid * G::F + f;
            const auto st = p.store.prep(g, g < p.n_fft);
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) p.store.put(st, j + G::TP * q, r.v[q]);
        }
    }
};

// ------------------------------------------------------------------------------------------
// Chirp-z transform on the unit circle, fully fused (M = G::L >= n_in + n_out - 1):
//   load x * pre (zero-padded to M) -> FFT_M -> * mult, conj -> FFT_M -> conj * post, first n_out
// Bluestein's algorithm is the case n_in = n_out = n, pre = post = chirp[i] = W_2n^(i^2 mod 2n)
// (src/twiddles.rs:25-57), mult = FFT_M of the wrapped conjugate chirp / M
// (src/algorithm/bluesteins_algorithm.rs:62-83).  The CZT plans (impl.inl, czt_tables) fill the
// same slots with the tables of an arbitrary arc.  REAL: the input rows are real (imaginary part 0;
// half the bytes read), the output is complex.
// ------------------------------------------------------------------------------------------
template <class G, bool SWAP, bool REAL = false>
struct BluesteinKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = 1;  // two FFTs inlined back to back: let it have the registers
    static constexpr int NP1 = Eng::NPHASE;
    static constexpr int NPHASE = 2 * NP1 - 1;
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::SMEM_ELEMS;
    struct Params {
        const void* in;      // rows of n_in samples: cx<T>, or T when REAL
        cx<T>* out;          // rows of n_out samples
        const cx<T>* pre;    // n_in entries
        const cx<T>* post;   // n_out entries
        const cx<T>* mult;   // M entries
        const cx<T>* tw;     // stage twiddles of the M-point FFT
        uint32_t n_in, n_out;
        uint64_t n_fft;
    };
    struct Regs { cx<T> v[G::E]; };

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        const uint64_t g = (uint64_t)bid * G::F + f;
        const bool ok = g < p.n_fft;
        if constexpr (P == 0) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                cx<T> v = mk<T>(0, 0);
                if (ok && e < p.n_in) {
                    if constexpr (REAL) {
                        v.x = ld_stream_r((const T*)p.in + g * (uint64_t)p.n_in + e);
                    } else {
                        v = ld_stream((const cx<T>*)p.in + g * (uint64_t)p.n_in + e);
                    }
                    if (SWAP) v = swap_ri(v);
                    v = cmul(v, ldg(p.pre + e));
                }
                r.v[q] = v;
            }
        }
        if constexpr (P < NP1) {
            Eng::template phase<P>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NP1 - 1) {
            // pointwise multiply + conjugate, then stage 0 of the second FFT straight from registers
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                r.v[q] = conj(cmul(r.v[q], ldg(p.mult + e)));
            }
            Eng::template phase<0>(tid, r.v, smem, p.tw);
        }
        if constexpr (P >= NP1) {
            Eng::template phase<P - NP1 + 1>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NPHASE - 1) {
            cx<T>* dst = p.out + g * (uint64_t)p.n_out;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                if (ok && e < p.n_out) {
                    cx<T> v = cmul(conj(r.v[q]), ldg(p.post + e));
                    st_stream(dst + e, SWAP ? swap_ri(v) : v);
                }
            }
        }
    }
};

// ------------------------------------------------------------------------------------------
// Rader, fully fused: prime length n = M + 1, M = G::L.
//   a[i] = x[gpow[i]]  (gpow[i] = g^(i+1) mod n);  A = FFT_M a;  X[0] = x0 + A[0];
//   b = conj(A .* D);  b[0] += conj(x0);  B = FFT_M b;  X[ginv[i]] = conj(B[i])
// (src/algorithm/raders_algorithm.rs:235-283; D = FFT_M(twiddle(g^-i)/M), :86-109)
// ------------------------------------------------------------------------------------------
template <class G, bool SWAP>
struct RaderKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = 1;  // two FFTs inlined back to back: let it have the registers
    static constexpr int NP1 = Eng::NPHASE;
    static constexpr int NPHASE = 2 * NP1 - 1;
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::SMEM_ELEMS;
    struct Params {
        const cx<T>* in;
        cx<T>* out;
        const uint32_t* gpow;  // M entries: g^(i+1) mod n
        const uint32_t* ginv;  // M entries: g^-(i+1) mod n
        const cx<T>* mult;     // M entries (D)
        const cx<T>* tw;
        uint32_t n;
        uint64_t n_fft;
    };
    struct Regs { cx<T> v[G::E]; cx<T> x0; };

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        const uint64_t g = (uint64_t)bid * G::F + f;
        const bool ok = g < p.n_fft;
        if constexpr (P == 0) {
            const cx<T>* src = p.in + g * (uint64_t)p.n;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                cx<T> v = mk<T>(0, 0);
                if (ok) {
                    v = src[ldg_u32(p.gpow + e)];
                    if (SWAP) v = swap_ri(v);
                }
                r.v[q] = v;
            }
            r.x0 = mk<T>(0, 0);
            if (ok && j == 0) {
                r.x0 = src[0];
                if (SWAP) r.x0 = swap_ri(r.x0);
            }
        }
        if constexpr (P < NP1) {
            Eng::template phase<P>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NP1 - 1) {
            if (ok && j == 0) {  // slot 0 of thread 0 is element 0 = sum of x[1..n)
                cx<T> dc = r.x0 + r.v[0];
                p.out[g * (uint64_t)p.n] = SWAP ? swap_ri(dc) : dc;
            }
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                r.v[q] = conj(cmul(r.v[q], ldg(p.mult + e)));
            }
            if (j == 0) r.v[0] = r.v[0] + conj(r.x0);
            Eng::template phase<0>(tid, r.v, smem, p.tw);
        }
        if constexpr (P >= NP1) {
            Eng::template phase<P - NP1 + 1>(tid, r.v, smem, p.tw);
        }
        if constexpr (P == NPHASE - 1) {
            cx<T>* dst = p.out + g * (uint64_t)p.n;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const uint32_t e = j + G::TP * q;
                if (ok) {
                    cx<T> v = conj(r.v[q]);
                    dst[ldg_u32(p.ginv + e)] = SWAP ? swap_ri(v) : v;
                }
            }
        }
    }
};

// ------------------------------------------------------------------------------------------
// SmoothKernel: one-pass Stockham FFT for lengths whose prime factors are all <= 31 and that have no compiled
// geometry (n <= SMOOTH_MAX).  The radix list is run-time data (the host planner factors n into stages of
// radix 31..11 / 7 / 5 / 3 / 16 / 8 / 4 / 2 -- the reference's RadixN does the same with 2..7 over a butterfly
// base taken from its hard-coded set 2..32, src/algorithm/radixn.rs:54-155, src/plan.rs:508-634); each stage is one pass over a ping-pong pair of
// shared-memory buffers, the first stage reads global memory and the last one writes it, both coalesced
// and in natural order (same index algebra as engine.h).  Slower per element than the compiled
// power-of-two geometries (no cross-stage register reuse, generic index arithmetic) but one pass over
// HBM and no padding to a power of two -- against Bluestein's two FFTs of 2-4x the length.
// ------------------------------------------------------------------------------------------
// RMAX = largest radix the instantiation carries: 16 drops the prime butterflies 11..31 from the stage switch, which are what push
// these kernels to 128 registers per thread (2 CTAs per SM); without them 3 CTAs fit
template <typename T, bool SWAP, int RMAX = 31>
struct SmoothKernel {
    using T_ = T;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = RMAX > 16 ? 2 : 3;
    static constexpr int MAX_STAGES = 8;
    static constexpr int NPHASE = MAX_STAGES;
    static constexpr size_t SMEM_BYTES = 0;  // run-time sized: Params::smem_bytes
    struct Params {
        const cx<T>* in;
        cx<T>* out;
        const cx<T>* tw;  // packed like the engine's: stage s >= 1 at tw_off[s], entry (r-1)*p + k = W_{pR}^{k r}
        uint64_t n_fft;
        uint32_t n, n_stages, f_per_cta, smem_bytes;
        uint32_t radix[MAX_STAGES];
        uint32_t tw_off[MAX_STAGES];
        FastDiv div_t[MAX_STAGES];  // by T_s = n / radix[s]
        FastDiv div_p[MAX_STAGES];  // by p_s = product of the radices before s
    };
    struct Regs {};

    template <int R>
    static B2_HD void stage(const Params& p, uint32_t bid, int tid, int s, cx<T>* smem) {
        const uint32_t n = p.n, F = p.f_per_cta;
        const uint32_t pp = p.div_p[s].d;  // product of the radices before stage s
        const uint32_t T_s = p.div_t[s].d;  // butterflies per transform = n / R
        const bool first = (s == 0), last = (s == (int)p.n_stages - 1);
        const cx<T>* src_buf = smem + (size_t)((s + 1) & 1) * F * n;  // stage s-1 wrote buffer (s-1)&1
        cx<T>* dst_buf = smem + (size_t)(s & 1) * F * n;
        const cx<T>* tws = p.tw + p.tw_off[s];
        for (uint32_t b = (uint32_t)tid; b < F * T_s; b += NT) {
            const uint32_t f = p.div_t[s].div(b), i = b - f * T_s;
            const uint64_t g = (uint64_t)bid * F + f;
            if (g >= p.n_fft) continue;
            const uint32_t k = i - p.div_p[s].div(i) * pp;
            cx<T> a[R];
            if (first) {
                const cx<T>* src = p.in + g * (uint64_t)n + i;
                B2_UNROLL
                for (int q = 0; q < R; ++q) {
                    cx<T> v = ld_stream(src + (size_t)q * T_s);
                    a[q] = SWAP ? swap_ri(v) : v;
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
                cx<T>* dst = p.out + g * (uint64_t)n + base;
                B2_UNROLL
                for (int m = 0; m < R; ++m) st_stream(dst + (size_t)m * pp, SWAP ? swap_ri(a[m]) : a[m]);
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
        switch (p.radix[P]) {
            case 2: stage<2>(p, bid, tid, P, smem); break;
            case 3: stage<3>(p, bid, tid, P, smem); break;
            case 4: stage<4>(p, bid, tid, P, smem); break;
            case 5: stage<5>(p, bid, tid, P, smem); break;
            case 7: stage<7>(p, bid, tid, P, smem); break;
            case 8: stage<8>(p, bid, tid, P, smem); break;
            case 16: stage<16>(p, bid, tid, P, smem); break;
            case 11: if constexpr (RMAX >= 11) stage<11>(p, bid, tid, P, smem); break;
            case 13: if constexpr (RMAX >= 13) stage<13>(p, bid, tid, P, smem); break;
            case 17: if constexpr (RMAX >= 17) stage<17>(p, bid, tid, P, smem); break;
            case 19: if constexpr (RMAX >= 19) stage<19>(p, bid, tid, P, smem); break;
            case 23: if constexpr (RMAX >= 23) stage<23>(p, bid, tid, P, smem); break;
            case 29: if constexpr (RMAX >= 29) stage<29>(p, bid, tid, P, smem); break;
            case 31: if constexpr (RMAX >= 31) stage<31>(p, bid, tid, P, smem); break;
            default: break;
        }
    }
};

// ------------------------------------------------------------------------------------------
// SmoothPassKernel: the two passes of a four-step over a COMPOSITE length N = N1 * N2 whose prime factors are all
// <= 31 (N1, N2 <= SMOOTH_MAX): the reference's MixedRadix (src/algorithm/mixed_radix.rs:128-158: columns FFT, twiddles,
// rows FFT, three transposes) with the transposes folded into strided loads / stores, run-time radix lists as in
// SmoothKernel.  Replaces Bluestein over a power-of-two four-step (four passes over 2-4x the data) for lengths
// such as 10000, 44100, 48000, 10^6.
//   MODE 1 (pass A): FFT g = (transform b, column c), g = b*N2 + c; element e at in[b*N + e*N2 + c]; the N1-point
//                    result k1 goes to work[b*N + k1*N2 + c].  Threads: column fastest (adjacent columns are
//                    adjacent in memory); shared memory [element][column].
//   MODE 2 (pass B): FFT g = (b, row k1), g = b*N1 + k1; element e at work[g*N2 + e], times W_N^(k1 e) (table
//                    [k1][n2], each entry rounded once); the N2-point result k2 goes to out[b*N + k2*N1 + k1].
//                    Threads: element fastest (contiguous loads) until the last stage, row fastest there
//                    (adjacent rows are adjacent in the output); shared memory [row][odd pitch].
// The body is SmoothPassBody; SmoothPassKernel is its R2D = 0 form, unchanged.  R2D (MODE 1 only, a compile-time variant that
// Real2dColumnKernel names) is the column pass of the 2-D real transforms, with the per-row real unpack / pack of real.h
// (M = W / 2) applied on the load:
//   R2D 1 (forward):  M + 1 output columns k of an [H][M + 1] spectrum from Z = the M-point row FFTs [H][M] of the real image:
//                     element e = E + W_W^k O, E = (Z[e][k mod M] + conj Z[e][(M-k) mod M]) / 2, O = (... - ...) / 2i
//   R2D 2 (inverse):  M output columns k of Z' [H][M] from the [H][M + 1] spectrum X, the row index of the partner reflected
//                     (IFFT_H of conj X[-k1][.] is conj of IFFT_H of X[k1][.]):
//                     element k1 = A + i conj(W_W^k) B, A / B = X[k1][k] +/- conj X[(H-k1) mod H][M-k]
//   R2D 3 (inverse, column 0 again; Real2dDcColumnKernel): the same element from the Hermitian parts of columns 0 and M, as
//                     numpy.fft.irfft2 keeps them; it overwrites the R2D 2 pass's column 0
// Column slot c of the `other` slots of an image holds column c / 2 (c even) or other - 1 - c / 2 (c odd), so the two columns a
// thread's load gathers are one warp's two contiguous runs, and lanes 2i and 2i + 1 read the same lines.  Store: [H][other].
// ------------------------------------------------------------------------------------------
template <typename T>
struct Real2dPassArgs {
    const cx<T>* wk;    // W_W^k, k = 0 .. M
    uint32_t half_w;    // M = W / 2
    uint32_t in_pitch;  // complex elements per input row: M (forward), M + 1 (inverse)
};
struct NoPassArgs {};
template <typename T, bool SW, int MODE, int RMAX, int R2D>
struct SmoothPassBody {
    static_assert(R2D == 0 || (MODE == 1 && SW == (R2D >= 2)), "the 2-D real column passes are MODE 1; the inverse ones run swapped");
    using T_ = T;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = RMAX > 16 ? 2 : 3;
    static constexpr int MAX_STAGES = 8;
    static constexpr int NPHASE = MAX_STAGES;
    static constexpr size_t SMEM_BYTES = 0;  // run-time sized: Params::smem_bytes
    struct Params : std::conditional_t<R2D != 0, Real2dPassArgs<T>, NoPassArgs> {
        const cx<T>* in;
        cx<T>* out;
        const cx<T>* tw;       // packed stage twiddles of this pass' length (layout as in SmoothKernel)
        const cx<T>* full_tw;  // MODE 2: W_N^(k1 n2), [N1][N2]
        uint64_t n_fft;        // FFTs of this launch (< 2^31)
        uint64_t NN;           // N = N1 * N2
        uint32_t n;            // length of this pass' FFTs
        uint32_t other;        // MODE 1: N2 (columns per transform);  MODE 2: N1 (rows per transform)
        uint32_t n_stages, f_per_cta, pitch, smem_bytes;
        uint32_t radix[MAX_STAGES];
        uint32_t tw_off[MAX_STAGES];
        FastDiv div_t[MAX_STAGES];  // by T_s = n / radix[s]
        FastDiv div_p[MAX_STAGES];  // by p_s = product of the radices before s
        FastDiv div_other, div_f;
        // --- variants of the same two passes (0 / null = the plain SmoothFourStep) ---
        // Good-Thomas (src/algorithm/good_thomas_algorithm.rs:144-248): N1, N2 coprime, no inter-pass twiddles (full_tw = null);
        // pass A reads x[crt1[n1] + crt2[n2] mod N] (the CRT map: n = n1 mod N1, n = n2 mod N2), pass B writes
        // X[(k1 N2 + k2 N1) mod N] (the Ruritanian map) -- the reference's reindex_input / reindex_output folded into the passes
        const uint32_t* crt1;  // N1 entries: n1 * N2 * (N2^-1 mod N1) mod N
        const uint32_t* crt2;  // N2 entries: n2 * N1 * (N1^-1 mod N2) mod N
        uint32_t gt;
        // large Rader / Bluestein plans over a smooth inner length M = N1 * N2 (the passes of LoadColsConv / StoreTransposedConv):
        //   MODE 1, conv 1: inner element i = e N2 + c comes from in[b n_outer + gather[i]]                       (Rader)
        //   MODE 1, conv 2: i < n_outer ? in[b n_outer + i] * chirp[i] : 0                                        (Bluestein)
        //   MODE 2, conv 1: end of inner FFT #1 -- out[b M + k] = conj(v * mult[k]) (+ Rader DC when x_in != null)
        //   MODE 2, conv 2: out[b n_outer + scatter[k]] = conj(v)                                                 (Rader)
        //   MODE 2, conv 3: k < n_outer: out[b n_outer + k] = conj(v) * chirp[k]                                  (Bluestein)
        uint32_t conv, n_outer;
        uint32_t swap_out;  // MODE 1 as a stand-alone column pass (2-D plans): re/im swap on the store too (inverse direction)
        const uint32_t* gather;
        const uint32_t* scatter;
        const cx<T>* chirp;
        const cx<T>* mult;
        const cx<T>* x_in;
        cx<T>* x_out;
    };
    struct Regs {};

    static B2_HD size_t sidx(const Params& p, uint32_t f, uint32_t e) {
        return MODE == 1 ? (size_t)e * p.f_per_cta + f : (size_t)f * p.pitch + e;
    }

    // elements between the output rows: `other`, except R2D 3 (one slot per image, column 0 of rows of M)
    static B2_HD uint32_t out_pitch(const Params& p) {
        if constexpr (R2D == 3) return p.half_w;
        else return p.other;
    }
    // 2-D real passes: the column a slot holds (partners adjacent, see above)
    static B2_HD uint32_t real2d_column(const Params& p, uint32_t c) { return (c & 1u) ? p.other - 1u - (c >> 1) : c >> 1; }
    // the R elements e = i + q T_s of column k of image b, unpacked (R2D 1) or packed (R2D 2) on the load -- real.h's arithmetic
    template <int R>
    static B2_HD void real2d_load(const Params& p, uint32_t b, uint32_t k, uint32_t i, uint32_t T_s, cx<T>* a) {
        const uint32_t M = p.half_w, H = p.n;
        const cx<T>* src = p.in + (uint64_t)b * H * p.in_pitch;
        if constexpr (R2D == 1) {
            const uint32_t ka = k == M ? 0u : k, kb = k == 0 ? 0u : M - k;
            const cx<T> w = ldg(p.wk + k);
            const T half = (T)0.5;
            B2_UNROLL
            for (int q = 0; q < R; ++q) {
                const cx<T>* row = src + (uint64_t)(i + (uint32_t)q * T_s) * M;
                const cx<T> zk = ldg(row + ka), zm = conj(ldg(row + kb));
                const cx<T> e = mk<T>((zk.x + zm.x) * half, (zk.y + zm.y) * half);
                const cx<T> d = mk<T>((zk.x - zm.x) * half, (zk.y - zm.y) * half);  // = i O
                const cx<T> o = mk<T>(d.y, -d.x);                                     // O = d / i
                a[q] = e + cmul(o, w);
            }
        } else if constexpr (R2D == 3) {
            // column 0 only (k = 0, W^0 = 1): the Hermitian parts (X[k1][0] + conj X[-k1][0]) / 2 and (X[-k1][M] + conj X[k1][M]) / 2,
            // then A + i B as above; equal to the R2D 2 element, bit for bit, when columns 0 and M are Hermitian
            const uint32_t P = p.in_pitch;  // M + 1
            const T half = (T)0.5;
            (void)k;
            B2_UNROLL
            for (int q = 0; q < R; ++q) {
                const uint32_t e = i + (uint32_t)q * T_s, er = e == 0 ? 0u : H - e;
                const cx<T> x0 = ldg(src + (uint64_t)e * P), xr = conj(ldg(src + (uint64_t)er * P));
                const cx<T> xm = conj(ldg(src + (uint64_t)er * P + M)), xn = ldg(src + (uint64_t)e * P + M);
                const cx<T> xk = mk<T>((x0.x + xr.x) * half, (x0.y + xr.y) * half), xh = mk<T>((xm.x + xn.x) * half, (xm.y + xn.y) * half);
                const cx<T> s = xk + xh, t = xk - xh;
                a[q] = swap_ri(s + mk<T>(-t.y, t.x));
            }
        } else {
            const uint32_t P = p.in_pitch;  // M + 1
            const cx<T> w = conj(ldg(p.wk + k));
            B2_UNROLL
            for (int q = 0; q < R; ++q) {
                const uint32_t e = i + (uint32_t)q * T_s, er = e == 0 ? 0u : H - e;
                const cx<T> xk = ldg(src + (uint64_t)e * P + k), xm = conj(ldg(src + (uint64_t)er * P + (M - k)));
                const cx<T> s = xk + xm, t = cmul(xk - xm, w);  // A, conj(W^k) B
                a[q] = swap_ri(s + mk<T>(-t.y, t.x));           // A + i conj(W^k) B, swapped for the inverse FFT
            }
        }
    }

    template <int R>
    static B2_HD void stage(const Params& p, uint32_t bid, int tid, int s, cx<T>* smem) {
        const uint32_t F = p.f_per_cta;
        const uint32_t pp = p.div_p[s].d;
        const uint32_t T_s = p.div_t[s].d;
        const bool first = (s == 0), last = (s == (int)p.n_stages - 1);
        const size_t half = (size_t)F * (MODE == 1 ? p.n : p.pitch);
        const cx<T>* src_buf = smem + (size_t)((s + 1) & 1) * half;
        cx<T>* dst_buf = smem + (size_t)(s & 1) * half;
        const cx<T>* tws = p.tw + p.tw_off[s];
        const bool f_fastest = (MODE == 1) || last;
        for (uint32_t idx = (uint32_t)tid; idx < F * T_s; idx += NT) {
            uint32_t f, i;
            if (f_fastest) {
                i = p.div_f.div(idx);
                f = idx - i * F;
            } else {
                f = p.div_t[s].div(idx);
                i = idx - f * T_s;
            }
            const uint64_t g = (uint64_t)bid * F + f;
            if (g >= p.n_fft) continue;
            const uint32_t b = p.div_other.div((uint32_t)g), c = (uint32_t)g - b * p.other;  // transform, column | row
            const uint32_t k = i - p.div_p[s].div(i) * pp;
            cx<T> a[R];
            if (first) {
                if constexpr (R2D != 0) {
                    real2d_load<R>(p, b, real2d_column(p, c), i, T_s, a);
                } else if (MODE == 1 && p.gt) {
                    const cx<T>* src = p.in + (uint64_t)b * p.NN;
                    const uint32_t o2 = ldg_u32(p.crt2 + c);
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) {
                        uint32_t o = ldg_u32(p.crt1 + i + (uint32_t)q * T_s) + o2;
                        if (o >= (uint32_t)p.NN) o -= (uint32_t)p.NN;
                        const cx<T> v = src[o];
                        a[q] = SW ? swap_ri(v) : v;
                    }
                } else if (MODE == 1 && p.conv) {
                    const cx<T>* src = p.in + (uint64_t)b * p.n_outer;
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) {
                        const uint32_t ii = (i + (uint32_t)q * T_s) * p.other + c;  // inner index e N2 + c
                        cx<T> v = mk<T>(0, 0);
                        if (p.conv == 1) {
                            v = src[ldg_u32(p.gather + ii)];
                            if (SW) v = swap_ri(v);
                        } else if (ii < p.n_outer) {
                            v = ld_stream(src + ii);
                            if (SW) v = swap_ri(v);
                            v = cmul(v, ldg(p.chirp + ii));
                        }
                        a[q] = v;
                    }
                } else if (MODE == 1) {
                    const cx<T>* src = p.in + (uint64_t)b * p.NN + c;
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) {
                        const cx<T> v = ld_cs(src + (uint64_t)(i + (uint32_t)q * T_s) * p.other);
                        a[q] = SW ? swap_ri(v) : v;
                    }
                } else if (p.full_tw == nullptr) {  // Good-Thomas: no inter-pass twiddles
                    const cx<T>* src = p.in + g * (uint64_t)p.n + i;
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) a[q] = ld_cs(src + (size_t)q * T_s);
                } else {
                    const cx<T>* src = p.in + g * (uint64_t)p.n + i;
                    const cx<T>* t = p.full_tw + (uint64_t)c * p.n + i;
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) a[q] = cmul(ld_cs(src + (size_t)q * T_s), ldg_stream(t + (size_t)q * T_s));
                }
            } else {
                B2_UNROLL
                for (int q = 0; q < R; ++q) a[q] = src_buf[sidx(p, f, i + (uint32_t)q * T_s)];
                B2_UNROLL
                for (int q = 1; q < R; ++q) a[q] = cmul(a[q], ldg(tws + (size_t)(q - 1) * pp + k));
            }
            Bfly<R, T>::run(a);
            const uint32_t base = (i - k) * R + k;
            if (last && MODE == 2 && p.gt) {
                cx<T>* dst = p.out + (uint64_t)b * p.NN;
                const uint32_t o1 = c * p.n;  // k1 N2
                B2_UNROLL
                for (int m = 0; m < R; ++m) {
                    uint32_t o = o1 + (base + (uint32_t)m * pp) * p.other;  // + k2 N1
                    if (o >= (uint32_t)p.NN) o -= (uint32_t)p.NN;
                    dst[o] = SW ? swap_ri(a[m]) : a[m];
                }
            } else if (last && MODE == 2 && p.conv) {
                B2_UNROLL
                for (int m = 0; m < R; ++m) {
                    const uint32_t kk = c + (base + (uint32_t)m * pp) * p.other;  // inner output index k1 + N1 k2
                    if (p.conv == 1) {
                        cx<T> w = conj(cmul(a[m], ldg(p.mult + kk)));
                        if (p.x_in != nullptr && kk == 0) {
                            cx<T> x0 = p.x_in[(uint64_t)b * p.n_outer];
                            if (SW) x0 = swap_ri(x0);
                            const cx<T> dc = x0 + a[m];
                            p.x_out[(uint64_t)b * p.n_outer] = SW ? swap_ri(dc) : dc;
                            w = w + conj(x0);
                        }
                        p.out[(uint64_t)b * p.NN + kk] = w;
                    } else if (p.conv == 2) {
                        const cx<T> w = conj(a[m]);
                        p.out[(uint64_t)b * p.n_outer + ldg_u32(p.scatter + kk)] = SW ? swap_ri(w) : w;
                    } else if (kk < p.n_outer) {
                        const cx<T> w = cmul(conj(a[m]), ldg(p.chirp + kk));
                        st_stream(p.out + (uint64_t)b * p.n_outer + kk, SW ? swap_ri(w) : w);
                    }
                }
            } else if (last) {
                cx<T>* dst;
                if constexpr (R2D != 0) dst = p.out + (uint64_t)b * p.NN + real2d_column(p, c);
                else dst = p.out + (uint64_t)b * p.NN + c;
                B2_UNROLL
                for (int m = 0; m < R; ++m) {
                    const cx<T> v = ((MODE == 2 && SW) || (MODE == 1 && p.swap_out)) ? swap_ri(a[m]) : a[m];
                    cx<T>* d = dst + (uint64_t)(base + (uint32_t)m * pp) * out_pitch(p);
                    if (MODE == 2) st_cs(d, v); else *d = v;  // pass A's output is re-read from L2 by pass B
                }
            } else {
                B2_UNROLL
                for (int m = 0; m < R; ++m) dst_buf[sidx(p, f, base + (uint32_t)m * pp)] = a[m];
            }
        }
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>* smem) {
        if (P >= (int)p.n_stages) return;
        switch (p.radix[P]) {
            case 2: stage<2>(p, bid, tid, P, smem); break;
            case 3: stage<3>(p, bid, tid, P, smem); break;
            case 4: stage<4>(p, bid, tid, P, smem); break;
            case 5: stage<5>(p, bid, tid, P, smem); break;
            case 7: stage<7>(p, bid, tid, P, smem); break;
            case 8: stage<8>(p, bid, tid, P, smem); break;
            case 16: stage<16>(p, bid, tid, P, smem); break;
            case 11: if constexpr (RMAX >= 11) stage<11>(p, bid, tid, P, smem); break;
            case 13: if constexpr (RMAX >= 13) stage<13>(p, bid, tid, P, smem); break;
            case 17: if constexpr (RMAX >= 17) stage<17>(p, bid, tid, P, smem); break;
            case 19: if constexpr (RMAX >= 19) stage<19>(p, bid, tid, P, smem); break;
            case 23: if constexpr (RMAX >= 23) stage<23>(p, bid, tid, P, smem); break;
            case 29: if constexpr (RMAX >= 29) stage<29>(p, bid, tid, P, smem); break;
            case 31: if constexpr (RMAX >= 31) stage<31>(p, bid, tid, P, smem); break;
            default: break;
        }
    }
};
template <typename T, bool SW, int MODE, int RMAX = 31>
struct SmoothPassKernel : SmoothPassBody<T, SW, MODE, RMAX, 0> {};
// R2D 1: forward (unpack, then the forward column FFT);  R2D 2: inverse (pack, then the inverse column FFT, re/im swapped)
template <typename T, int R2D, int RMAX>
struct Real2dColumnKernel : SmoothPassBody<T, R2D == 2, 1, RMAX, R2D> {};
// R2D 3: the inverse column pass again, for column 0 alone, after Real2dColumnKernel<T, 2>: numpy.fft.irfft2's last-axis irfft keeps
// only the Hermitian parts of columns 0 and M, which the plain pack does not separate.  One slot (column 0) per image.
template <typename T, int RMAX>
struct Real2dDcColumnKernel : SmoothPassBody<T, true, 1, RMAX, 3> {};

// ------------------------------------------------------------------------------------------
// SmoothConvKernel: a whole convolution-based transform in ONE CTA pass over a SMOOTH inner length M (prime factors
// <= 31, run-time radix list as in SmoothKernel):
//   MODE_RADER      prime p = M + 1 (src/algorithm/raders_algorithm.rs:235-283): gather by g^(i+1) -> FFT_M -> DC, x D, conj
//                   -> FFT_M -> conj, scatter by g^-(i+1).  This is what makes every "easy" prime (p - 1 smooth -- the
//                   reference's rule, src/plan.rs:129,636-664) a one-pass plan instead of a Bluestein over 2-4x the data.
//                   With an OUTER radix r0 > 1 the transform length is n = r0 * p and the kernel is the reference's
//                   MixedRadix{r0 x Rader(p)} (src/plan.rs:412-425; e.g. 1234 = 2 x Rader(617), SURVEY 3.1) fused: virtual
//                   transform (t, k1) runs Rader on u[n2] = W_n^(n2 k1) * sum_n1 x_t[n1 p + n2] W_r0^(n1 k1), its result k2
//                   lands on X_t[k1 + r0 k2].
//   MODE_BLUESTEIN  any n with 2n - 1 <= M (src/algorithm/bluesteins_algorithm.rs:100-136): x * chirp, zero pad -> FFT_M
//                   -> x mult, conj -> FFT_M -> conj * chirp; lets M be the smallest 2^a 3^b 5^c 7^d instead of the next
//                   power of two (the idea of src/plan.rs:649-657 and src/avx/avx_planner.rs:945-994).
// 2 S steps (S = stages of the M-point FFT) over a ping-pong pair of shared-memory buffers, a CTA barrier between steps;
// step 0 reads global memory, step S - 1 does the DC bookkeeping, step S applies the pointwise multiply on its loads,
// step 2 S - 1 writes global memory.  The step index is run-time data (run_kernel_loop): 14 butterfly bodies per
// precision instead of 14 x 16.
// ------------------------------------------------------------------------------------------
template <typename T, bool SW, int RMAX = 31>
struct SmoothConvKernel {
    using T_ = T;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = RMAX > 16 ? 2 : 3;
    static constexpr int MAX_STAGES = 8;
    static constexpr int NPHASE = 2 * MAX_STAGES;  // CPU replay: phase<P> = step P
    static constexpr size_t SMEM_BYTES = 0;        // run-time sized: Params::smem_bytes
    static constexpr uint32_t MODE_RADER = 0, MODE_BLUESTEIN = 1;
    struct Params {
        const cx<T>* in;
        cx<T>* out;
        const cx<T>* tw;        // packed stage twiddles of the M-point FFT (layout as in SmoothKernel)
        const cx<T>* mult;      // M entries
        const uint32_t* gpow;   // Rader: g^(i+1) mod p
        const uint32_t* ginv;   // Rader: g^-(i+1) mod p
        const cx<T>* chirp;     // Bluestein: W_2n^(i^2), n entries
        const cx<T>* otw;       // r0 > 1: W_n^(n2 k1), [k1][n2] (r0 x p entries)
        const cx<T>* w_r0;      // r0 > 1: W_r0^j, r0 entries
        uint64_t n_fft;         // transforms of length n in this launch
        uint32_t n;             // transform length (Rader: r0 * p)
        uint32_t p;             // Rader: the prime (M + 1)
        uint32_t M, r0, mode;
        uint32_t n_stages, f_per_cta, smem_bytes;  // f_per_cta = VIRTUAL transforms per CTA (a multiple of r0)
        uint32_t radix[MAX_STAGES];
        uint32_t tw_off[MAX_STAGES];
        FastDiv div_t[MAX_STAGES];  // by T_s = M / radix[s]
        FastDiv div_p[MAX_STAGES];  // by p_s = product of the radices before s
        FastDiv div_r0;
    };
    struct Regs {};

    static B2_HD cx<T> ld_in(const Params& p, uint64_t off) {
        const cx<T> v = ld_stream(p.in + off);
        return SW ? swap_ri(v) : v;
    }
    // Rader input of virtual transform (t, k1) at n2: the outer radix-r0 butterfly and its twiddle, folded into the load
    static B2_HD cx<T> u_at(const Params& p, uint64_t t, uint32_t k1, uint32_t n2) {
        const uint64_t base = t * (uint64_t)p.n + n2;
        if (p.r0 == 1) return ld_in(p, base);
        cx<T> acc = ld_in(p, base);
        uint32_t j = 0;
        for (uint32_t n1 = 1; n1 < p.r0; ++n1) {
            j += k1;
            if (j >= p.r0) j -= p.r0;
            acc = acc + cmul(ld_in(p, base + (uint64_t)n1 * p.p), ldg(p.w_r0 + j));
        }
        return k1 ? cmul(acc, ldg(p.otw + (size_t)k1 * p.p + n2)) : acc;
    }

    template <int R>
    static B2_HD void stage(const Params& p, uint32_t bid, int tid, uint32_t step, cx<T>* smem) {
        const uint32_t S = p.n_stages, M = p.M, F = p.f_per_cta;
        const bool second = step >= S;
        const uint32_t s = second ? step - S : step;
        const bool first_s = (s == 0), last_s = (s == S - 1);
        const uint32_t pp = p.div_p[s].d, T_s = p.div_t[s].d;
        const cx<T>* src_buf = smem + (size_t)((step + 1) & 1) * F * M;
        cx<T>* dst_buf = smem + (size_t)(step & 1) * F * M;
        cx<T>* u0s = smem + (size_t)2 * F * M;  // Rader: u[0] of every virtual transform of the CTA
        const cx<T>* tws = p.tw + p.tw_off[s];
        const bool rader = p.mode == MODE_RADER;
        for (uint32_t b = (uint32_t)tid; b < F * T_s; b += NT) {
            const uint32_t f = p.div_t[s].div(b), i = b - f * T_s;
            const uint64_t gv = (uint64_t)bid * F + f;
            const uint64_t t = p.r0 == 1 ? gv : (uint64_t)p.div_r0.div((uint32_t)gv);
            if (t >= p.n_fft) continue;
            const uint32_t k1 = (uint32_t)(gv - t * p.r0);
            const uint32_t k = i - p.div_p[s].div(i) * pp;
            cx<T> a[R];
            if (first_s && !second) {
                B2_UNROLL
                for (int q = 0; q < R; ++q) {
                    const uint32_t idx = i + (uint32_t)q * T_s;
                    if (rader) {
                        a[q] = u_at(p, t, k1, ldg_u32(p.gpow + idx));
                    } else {
                        a[q] = idx < p.n ? cmul(ld_in(p, t * (uint64_t)p.n + idx), ldg(p.chirp + idx)) : mk<T>(0, 0);
                    }
                }
                if (rader && i == 0) u0s[f] = u_at(p, t, k1, 0);  // (the same thread owns output 0 of every stage)
            } else {
                const cx<T>* src = src_buf + (size_t)f * M + i;
                B2_UNROLL
                for (int q = 0; q < R; ++q) a[q] = src[(size_t)q * T_s];
                if (first_s) {  // first stage of the second FFT: pointwise multiply + conjugate on the way in
                    B2_UNROLL
                    for (int q = 0; q < R; ++q) a[q] = conj(cmul(a[q], ldg(p.mult + i + (uint32_t)q * T_s)));
                    if (rader && i == 0) a[0] = a[0] + conj(u0s[f]);
                } else {
                    B2_UNROLL
                    for (int q = 1; q < R; ++q) a[q] = cmul(a[q], ldg(tws + (size_t)(q - 1) * pp + k));
                }
            }
            Bfly<R, T>::run(a);
            const uint32_t base = (i - k) * R + k;
            if (last_s && second) {
                if (rader) {
                    cx<T>* dst = p.out + t * (uint64_t)p.n + k1;
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) {
                        const cx<T> v = conj(a[m]);
                        dst[(size_t)p.r0 * ldg_u32(p.ginv + base + (uint32_t)m * pp)] = SW ? swap_ri(v) : v;
                    }
                } else {
                    cx<T>* dst = p.out + t * (uint64_t)p.n;
                    B2_UNROLL
                    for (int m = 0; m < R; ++m) {
                        const uint32_t o = base + (uint32_t)m * pp;
                        if (o < p.n) {
                            const cx<T> v = cmul(conj(a[m]), ldg(p.chirp + o));
                            st_stream(dst + o, SW ? swap_ri(v) : v);
                        }
                    }
                }
            } else {
                cx<T>* dst = dst_buf + (size_t)f * M + base;
                B2_UNROLL
                for (int m = 0; m < R; ++m) dst[(size_t)m * pp] = a[m];
                if (last_s && rader && i == 0) {  // X[0] = u[0] + sum of the rest (raders_algorithm.rs:252-262)
                    const cx<T> dc = u0s[f] + a[0];
                    p.out[t * (uint64_t)p.n + k1] = SW ? swap_ri(dc) : dc;
                }
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
            case 11: if constexpr (RMAX >= 11) stage<11>(p, bid, tid, st, smem); break;
            case 13: if constexpr (RMAX >= 13) stage<13>(p, bid, tid, st, smem); break;
            case 17: if constexpr (RMAX >= 17) stage<17>(p, bid, tid, st, smem); break;
            case 19: if constexpr (RMAX >= 19) stage<19>(p, bid, tid, st, smem); break;
            case 23: if constexpr (RMAX >= 23) stage<23>(p, bid, tid, st, smem); break;
            case 29: if constexpr (RMAX >= 29) stage<29>(p, bid, tid, st, smem); break;
            case 31: if constexpr (RMAX >= 31) stage<31>(p, bid, tid, st, smem); break;
            default: break;
        }
    }
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>* smem) { step(p, bid, tid, (uint32_t)P, smem); }
};

// ------------------------------------------------------------------------------------------
// Persistent, software-pipelined one-pass kernels (contiguous tiles).
//
// A tile = F whole FFTs that are contiguous in global memory (Direct: F transforms; four-step pass B:
// F rows of the [k1][n2] intermediate).  CTAs are persistent (grid = SMs x resident CTAs) and stride
// over the tiles; while tile i is transformed out of shared-memory buffer i&1, ONE thread has already
// queued tile i+1 into the other buffer with a single TMA bulk copy (cp.async.bulk -> UBLKCP) that
// completes on an mbarrier.  The signal therefore never passes through the LSU's global-load queue
// (lg_throttle / mio_throttle are the top stalls of the LDG-based kernels) and the copy
// of the next tile overlaps all of the current tile's butterflies.  The buffer that received the
// dense tile is then reused, in place, as the padded exchange buffer of the stages.
//   phase 0     : dense tile -> registers  (+ Xform: re/im swap, or the inter-pass twiddle table)
//   phase 1..   : the engine's phases
//   last phase  : Store functor straight from registers (coalesced)
// ------------------------------------------------------------------------------------------
template <typename T, bool SWAP>
struct XformSwap {  // Direct plans: optional re<->im swap of an inverse plan
    struct St {};
    B2_HD St prep(uint64_t) const { return St{}; }
    B2_HD cx<T> apply(const St&, int, cx<T> v) const { return SWAP ? swap_ri(v) : v; }
};
template <typename T>
struct XformRowTw {  // four-step pass B: times W_N^(k1*n2), table [k1][n2]
    const cx<T>* tw;
    uint32_t len, lg1;
    struct St { const cx<T>* t; };
    B2_HD St prep(uint64_t g) const { return St{tw + (g & ((1ull << lg1) - 1)) * (uint64_t)len}; }
    B2_HD cx<T> apply(const St& s, int e, cx<T> v) const { return cmul(v, ldg_stream(s.t + e)); }
};

template <class G, Map M1, class Xform, class Store>
struct PipeKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, M1>;
    static constexpr int NT = G::NT;
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, G::E);
    static constexpr int NPHASE = Eng::NPHASE + 1;
    static constexpr size_t BUF_ELEMS = ((size_t)G::F * G::LP + 15) / 16 * 16;  // >= F*L, 128-byte multiple
    static constexpr size_t BUF_BYTES = BUF_ELEMS * sizeof(cx<T>);
    static constexpr size_t SMEM_BYTES = 2 * BUF_BYTES + 16;  // two buffers + two mbarriers
    static_assert(G::NS >= 2, "single-stage sizes use the plain kernels");
    struct Params {
        const cx<T>* in;   // tiles are contiguous: tile i starts at in + i*F*L
        Xform xform;
        Store store;
        const cx<T>* tw;
        uint64_t n_fft;
        uint32_t n_items;
    };
    struct Regs { cx<T> v[G::E]; };

    static B2_HD const cx<T>* fetch_src(const Params& p, uint32_t item) { return p.in + (uint64_t)item * G::F * G::L; }
    static B2_HD uint32_t fetch_bytes(const Params& p, uint32_t item) {
        const uint64_t first = (uint64_t)item * G::F;
        const uint64_t valid = (p.n_fft - first < (uint64_t)G::F) ? (p.n_fft - first) : (uint64_t)G::F;
        return (uint32_t)(valid * G::L * sizeof(cx<T>));
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t item, int tid, Regs& r, cx<T>* buf) {
        if constexpr (P == 0) {
            int f, j;
            tid_to_fj<G, JF>(tid, f, j);
            uint64_t g = (uint64_t)item * G::F + f;
            const auto st = p.xform.prep(g < p.n_fft ? g : p.n_fft - 1);
            const cx<T>* src = buf + f * G::L + j;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) r.v[q] = p.xform.apply(st, j + G::TP * q, src[G::TP * q]);
        } else {
            Eng::template phase<P - 1>(tid, r.v, buf, p.tw);
        }
        if constexpr (P == NPHASE - 1) {
            int f, j;
            Eng::out_owner(tid, f, j);
            const uint64_t g = (uint64_t)item * G::F + f;
            const auto st = p.store.prep(g, g < p.n_fft);
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) p.store.put(st, j + G::TP * q, r.v[q]);
        }
    }
};

// ------------------------------------------------------------------------------------------
// Four-step passes whose tiles move between global and shared memory through TMA (tensor maps).
//
// Profile of the LDG/STG passes: top stall = lg_throttle.  A warp request that touches a
// 64-byte run in each of four 128-byte lines (8-column tiles of 8-byte elements) costs the L1TEX tag stage four
// passes, and three of the four global accesses of the two passes are of that shape.  Here the LSU issues NO
// global access for the signal: one thread asks the TMA unit for the whole [L rows x F columns] box (pass A in /
// out, pass B out; pass B in is one contiguous bulk copy), the tile lands dense in shared memory
// (element (e, f) at e*F + f, read / written by "f fastest" threads as 256 contiguous bytes per warp: conflict
// free), and the same buffer is then reused, in place, as the padded exchange buffer of the stages and finally
// as the dense staging tile of the outgoing TMA store.
//   phase 0            dense tile -> registers (+ re/im swap of an inverse plan | x inter-pass twiddle)
//   phase 1 .. NS*2-1  the engine's phases; the last one also writes the dense output tile
//   last phase         one thread: TMA store of the tile (cp.async.bulk.tensor ... bulk_group) and its drain
// ROLE 0 = pass A (strided column tile in, same box out to the workspace), ROLE 1 = pass B (F contiguous rows in,
// transposed box out: out[b][k2][k1]).
// ------------------------------------------------------------------------------------------
template <class G> struct RL_last_pow2 {
    static constexpr int R = G::RL::get(G::NS - 1);
    static constexpr bool value = R >= 8 && (R & (R - 1)) == 0;
};
// TILED (fused.h): the workspace ring is TILE-MAJOR -- transform slot = TA dense pass-A tiles [tile][k1][f], 64 KiB each.
//   ROLE 0, TILED != 0: the results go from the registers straight to the ring with fully coalesced 8-byte stores (the
//       dense tile IS the memory layout), so the shared-memory buffer is dead after the last exchange read and pass-A tiles
//       never touch the TMA store path (49 GB/s per SM, measured: the scarce resource of the fused kernel);
//   ROLE 1, TILED = F of pass A: the tile (F rows x L columns) is gathered by one 4-D tensor copy [all TA tiles][F rows]
//       [FO columns] and lands as [tile][row][column-in-tile]; phase 0 reads it with that index map.
//   ROLE 1, DOUT: the finished rows go from the registers straight to the caller's output (runs of F consecutive k1, 64-256 bytes)
//       instead of through the dense tile and a TMA store: the shared-memory stage is free after the last exchange read and the SM's
//       TMA unit only carries the three other transfers of a tile pair (fused.h, B200FFT_FUSED_BDIRECT)
template <class G, Map M0, Map M1, int ROLE, bool SW, int TILED = 0, bool DOUT = false>
struct TmaTileKernel {
    using T = typename G::T;
    using Eng = Engine<G, M0, M1>;
    static constexpr int NT = G::NT;
#if defined(B2_TMA_MINB)
    static constexpr int MIN_BLOCKS = (G::E >= 32 && sizeof(T) == 4) ? B2_TMA_MINB : default_min_blocks(G::NT, G::E);
#else
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, G::E);
#endif
    static constexpr int NPHASE = Eng::NPHASE + 2;
    static constexpr size_t TILE_ELEMS = (size_t)G::F * G::L;
    static constexpr size_t BUF_ELEMS = ((TILE_ELEMS > (size_t)G::SMEM_ELEMS ? TILE_ELEMS : (size_t)G::SMEM_ELEMS) + 15) / 16 * 16;
    static constexpr size_t SMEM_BYTES = BUF_ELEMS * sizeof(cx<T>);
    static constexpr uint32_t TILE_BYTES = (uint32_t)(TILE_ELEMS * sizeof(cx<T>));
    static constexpr int BOX_ROWS = G::L < 256 ? G::L : 256;
    static constexpr int NBOX = G::L / BOX_ROWS;
    static_assert(G::NS >= 2, "single-stage sizes use the plain kernels");
    struct Params {
        TMap map_in;   // ROLE 0: the user's input as [transform][N1 rows][N2 columns]
        TMap map_out;  // ROLE 0: workspace, same shape;  ROLE 1: the user's output as [transform][N2 rows][N1 columns]
        const cx<T>* in;       // what map_in describes (ROLE 1: the workspace, source of the bulk copy)
        cx<T>* out;            // what map_out describes
        const cx<T>* tw;       // packed stage twiddles
        const cx<T>* full_tw;  // ROLE 1: inter-pass twiddles [N1][N2]
        uint64_t n_fft;        // FFTs of this launch (a whole number of tiles)
        uint32_t lgN, lg_other;  // ROLE 0: lg_other = log2 N2;  ROLE 1: lg_other = log2 N1
        uint32_t z_in, z_out;    // transform index of this launch's first transform inside `in` / `out`
        uint32_t discard;        // ROLE 1: drop the consumed workspace rows from L2 without write-back
        const void* pf;          // ROLE 1, opt-in (B200FFT_PREFETCH=1): input of the NEXT chunk of this stream; every CTA asks
        uint32_t pf_bytes;       //   L2 to fetch its pf_bytes share of it while this pass is still writing output
        const cx<T>* tw_lo;      // ROLE 1, optional: two-level inter-pass twiddles W_N^m = tw_hi[m >> 10] * tw_lo[m & 1023] (tw_lo[i] =
        const cx<T>* tw_hi;      //   W_N^i, tw_hi[h] = W_N^(1024 h)): 16 KiB that stay in L1 instead of an N-entry table streamed from L2
        uint32_t ring_w;         // fused single-launch plans (fused.h): the workspace is a ring of ring_w transform slots --
                                 //   ROLE 0 stores to / ROLE 1 loads from slot (transform mod ring_w); 0 = plain chunk workspace
    };
    static constexpr bool DIRECT_OUT = (ROLE == 0 && TILED != 0) || (ROLE == 1 && DOUT);  // registers -> tile-major ring | output
    static constexpr int FO = (ROLE == 1 && TILED > 0) ? TILED : 1;  // ROLE 1: columns per pass-A tile
    static constexpr int TA = G::L / FO;                             // ROLE 1: pass-A tiles per transform
    static constexpr int TBOX = TA < 256 ? TA : 256;                 // tiles per tensor copy
    static constexpr bool TILED_IN = (ROLE == 1 && TILED > 0);
    static_assert(!TILED_IN || (G::L % FO == 0 && TA % TBOX == 0), "tile-major ring geometry");
    // index of element (row f, column n2 = j + TP q) inside the gathered tile = base(f, j) + tiled_off(q)
    static B2_HD int tiled_base(int f, int j) {
        if constexpr (G::TP % FO == 0) return ((j / FO) * G::F + f) * FO + (j % FO);
        else return f * FO + j;
    }
    static constexpr int tiled_off(int q) {
        if (G::TP % FO == 0) return q * G::TP * G::F;
        return ((G::TP * q) / FO) * G::F * FO + (G::TP * q) % FO;
    }
    static_assert(!TILED_IN || G::TP % FO == 0 || FO % G::TP == 0, "powers of two");
    // slab (transform slot) a tile is read from / written to
    static B2_HD uint32_t zin(const Params& p, uint32_t b) { return (ROLE == 1 && p.ring_w) ? (p.z_in + b) % p.ring_w : p.z_in + b; }
    static B2_HD uint32_t zout(const Params& p, uint32_t b) { return (ROLE == 0 && p.ring_w) ? (p.z_out + b) % p.ring_w : p.z_out + b; }
    // tables fetched while the tile is in flight (f32, two-stage tiles): the last stage's twiddles (into L1 only: held in
    // registers through phases 0 and 1 they made the fused kernel's consumers spill) and, for pass B, the row's
    // inter-pass twiddles -- the round-1 capture of these kernels had long_scoreboard (table loads issued right before
    // their use) as the top stall
    static constexpr bool PRE = (G::NS == 2) && sizeof(T) == 4 && ((RL_last_pow2<G>::value));
    static constexpr int LGE = ilog2_c(G::E);
    struct Regs {
        cx<T> v[G::E];
        cx<T> rw[LGE + 1];  // ROLE 1: W^(k1 j), W^(k1 TP 2^i)
    };
    struct Where { uint32_t b, c0; };  // transform of the launch, first column (ROLE 0) / first row (ROLE 1) of the tile
    static B2_HD void prefetch(const Params& p, uint32_t bid, int tid, Regs& r) {
        if constexpr (PRE) {
            int f, j;
            Eng::out_owner(tid, f, j);
            Eng::template prefetch_tw<G::NS - 1>(j, p.tw);
            if (ROLE == 1) {
                const Where w = where(p, bid);
                Eng::template owner<0>(tid, f, j);
                if (p.tw_lo != nullptr) {
                    // W_N^(k1 x) from two L1-resident tables (one more rounding than the full table, no trip to L2)
                    const uint32_t k1 = w.c0 + (uint32_t)f, mask = (1u << p.lgN) - 1u;
                    auto tw2 = [&](uint32_t x) -> cx<T> {
                        const uint32_t m = (k1 * x) & mask;
                        return cmul(ldg(p.tw_hi + (m >> 10)), ldg(p.tw_lo + (m & 1023u)));
                    };
                    r.rw[0] = tw2((uint32_t)j);
                    B2_UNROLL
                    for (int l = 0; l < LGE; ++l) r.rw[l + 1] = tw2((uint32_t)(G::TP * (1 << l)));
                } else {
                    const cx<T>* t = p.full_tw + (uint64_t)(w.c0 + f) * G::L;
                    r.rw[0] = ldg_stream(t + j);
                    B2_UNROLL
                    for (int l = 0; l < LGE; ++l) r.rw[l + 1] = ldg_stream(t + G::TP * (1 << l));
                }
            }
        }
    }
    static B2_HD Where where(const Params& p, uint32_t bid) {
        const uint64_t g0 = (uint64_t)bid * G::F;
        return Where{(uint32_t)(g0 >> p.lg_other), (uint32_t)(g0 & ((1ull << p.lg_other) - 1))};
    }

#if defined(__CUDACC__)
    // pol != 0: an L2 eviction-priority policy (createpolicy) for the tile's lines
    static B2_D void issue_load(const Params& p, uint32_t bid, cx<T>* buf, uint64_t* bar, unsigned long long pol = 0) {
        const Where w = where(p, bid);
        tma::mbar_arrive_expect_tx(bar, TILE_BYTES);
        if (ROLE == 0) {
            B2_UNROLL
            for (int k = 0; k < NBOX; ++k) {
                if (pol)
                    tma::tensor_g2s_3d_hint(buf + (size_t)k * BOX_ROWS * G::F, &p.map_in, (int)(2 * w.c0), k * BOX_ROWS, (int)zin(p, w.b), bar, pol);
                else
                    tma::tensor_g2s_3d(buf + (size_t)k * BOX_ROWS * G::F, &p.map_in, (int)(2 * w.c0), k * BOX_ROWS, (int)zin(p, w.b), bar);
            }
        } else if constexpr (TILED_IN) {
            B2_UNROLL
            for (int k = 0; k < TA / TBOX; ++k) {
                if (pol)
                    tma::tensor_g2s_4d_hint(buf + (size_t)k * TBOX * G::F * FO, &p.map_in, 0, (int)w.c0, k * TBOX, (int)zin(p, w.b), bar, pol);
                else
                    tma::tensor_g2s_4d(buf + (size_t)k * TBOX * G::F * FO, &p.map_in, 0, (int)w.c0, k * TBOX, (int)zin(p, w.b), bar);
            }
        } else {
            if (pol)
                tma::bulk_g2s_hint(buf, p.in + ((uint64_t)zin(p, w.b) << p.lgN) + (uint64_t)w.c0 * G::L, TILE_BYTES, bar, pol);
            else
                tma::bulk_g2s(buf, p.in + ((uint64_t)zin(p, w.b) << p.lgN) + (uint64_t)w.c0 * G::L, TILE_BYTES, bar);
            if (p.pf != nullptr && p.pf_bytes) tma::bulk_prefetch_l2(static_cast<const char*>(p.pf) + (uint64_t)bid * p.pf_bytes, p.pf_bytes);
        }
    }
    // one thread: TMA store of the finished dense tile (joins the thread's bulk group; the caller commits / waits)
    static B2_D void issue_store(const Params& p, uint32_t bid, const cx<T>* buf, unsigned long long pol = 0) {
        const Where w = where(p, bid);
        B2_UNROLL
        for (int k = 0; k < NBOX; ++k) {
            if (pol)
                tma::tensor_s2g_3d_hint(&p.map_out, (int)(2 * w.c0), k * BOX_ROWS, (int)zout(p, w.b), buf + (size_t)k * BOX_ROWS * G::F, pol);
            else
                tma::tensor_s2g_3d(&p.map_out, (int)(2 * w.c0), k * BOX_ROWS, (int)zout(p, w.b), buf + (size_t)k * BOX_ROWS * G::F);
        }
    }
#endif

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* buf) {
        if constexpr (P == 0) {
            const Where w = where(p, bid);
#if !defined(__CUDA_ARCH__)
            prefetch(p, bid, tid, r);  // CPU replay (the device does it while the tile is in flight)
            if (tid == 0) {  // CPU replay: the TMA load is a copy
                if (ROLE == 0) {
                    const cx<T>* src = p.in + ((uint64_t)zin(p, w.b) << p.lgN) + w.c0;
                    for (int e = 0; e < G::L; ++e)
                        for (int f = 0; f < G::F; ++f) buf[e * G::F + f] = src[((uint64_t)e << p.lg_other) + f];
                } else if constexpr (TILED_IN) {
                    const cx<T>* src = p.in + ((uint64_t)zin(p, w.b) << p.lgN);
                    for (int t = 0; t < TA; ++t)
                        for (int f = 0; f < G::F; ++f)
                            for (int c = 0; c < FO; ++c) buf[((size_t)t * G::F + f) * FO + c] = src[(size_t)t * TILE_ELEMS + (size_t)(w.c0 + f) * FO + c];
                } else {
                    const cx<T>* src = p.in + ((uint64_t)zin(p, w.b) << p.lgN) + (uint64_t)w.c0 * G::L;
                    for (size_t i = 0; i < TILE_ELEMS; ++i) buf[i] = src[i];
                }
            }
#endif
            int f, j;
            Eng::template owner<0>(tid, f, j);
            if (ROLE == 0) {
                const cx<T>* src = buf + (size_t)j * G::F + f;
                B2_UNROLL
                for (int q = 0; q < G::E; ++q) {
                    const cx<T> v = src[(size_t)G::TP * q * G::F];
                    r.v[q] = SW ? swap_ri(v) : v;
                }
            } else {
                // element (row f, column j + TP q): row-major tile, or [pass-A tile][row][column-in-tile] when gathered from the
                // tile-major ring
                const cx<T>* src = TILED_IN ? buf + tiled_base(f, j) : buf + (size_t)f * G::L + j;
                auto at = [&](int q) -> cx<T> { return TILED_IN ? src[tiled_off(q)] : src[G::TP * q]; };
                const cx<T>* t = p.full_tw + (uint64_t)(w.c0 + f) * G::L + j;
#if defined(B2_TWROW_FEW)
                if constexpr (sizeof(T) == 4) {
                    cx<T> wq[G::E];
                    const cx<T> a = PRE ? r.rw[0] : ldg_stream(t);
                    B2_UNROLL
                    for (int q = 1, l = 1; q < G::E; q <<= 1, ++l) wq[q] = PRE ? r.rw[l] : ldg_stream(t - j + G::TP * q);
                    r.v[0] = cmul(at(0), a);
                    // each product twiddle next to its first use: the upper half (q >= E/2) is never a factor, so it dies at once
                    B2_UNROLL
                    for (int q = 1; q < G::E; ++q) {
                        if (q & (q - 1)) wq[q] = cmul(wq[hibit(q)], wq[q - hibit(q)]);
                        r.v[q] = cmul(at(q), cmul(a, wq[q]));
                    }
                } else
#endif
                {
                    B2_UNROLL
                    for (int q = 0; q < G::E; ++q) r.v[q] = cmul(at(q), ldg_stream(t + G::TP * q));
                }
            }
        } else if constexpr (P < NPHASE - 1) {
            if constexpr (P == 1 && ROLE == 1) {
                if (p.discard) {  // the tile is in shared memory / registers: its workspace rows are dead
                    const Where w = where(p, bid);
                    if constexpr (TILED_IN) {
                        // TA chunks of F rows x FO columns (contiguous), one per pass-A tile; whole 128-byte lines only
                        constexpr uint32_t CHUNK = (uint32_t)(G::F * FO * sizeof(cx<T>));
                        if constexpr (CHUNK % 128 == 0) {
                            constexpr uint32_t LPC = CHUNK / 128;
                            const char* base = reinterpret_cast<const char*>(p.in + ((uint64_t)zin(p, w.b) << p.lgN) + (uint64_t)w.c0 * FO);
                            for (uint32_t l = (uint32_t)tid; l < TILE_BYTES / 128; l += (uint32_t)G::NT)
                                l2_discard_line(base + (size_t)(l / LPC) * TILE_BYTES + (size_t)(l % LPC) * 128);
                        }
                    } else {
                        const char* base = reinterpret_cast<const char*>(p.in + ((uint64_t)zin(p, w.b) << p.lgN) + (uint64_t)w.c0 * G::L);
                        for (uint32_t l = (uint32_t)tid; l < TILE_BYTES / 128; l += (uint32_t)G::NT) l2_discard_line(base + (size_t)l * 128);
                    }
                }
            }
            Eng::template phase<P - 1>(tid, r.v, buf, p.tw);
            if constexpr (P == NPHASE - 2) {
                int f, j;
                Eng::out_owner(tid, f, j);
                if constexpr (ROLE == 1 && DOUT) {
                    // row k1 = c0 + f, output k2 = j + TP q -> out[b N + k2 N1 + k1]: consecutive threads = consecutive k1
                    const Where w = where(p, bid);
                    cx<T>* dst = p.out + ((uint64_t)zout(p, w.b) << p.lgN) + w.c0 + f + ((size_t)j << p.lg_other);
                    B2_UNROLL
                    for (int q = 0; q < G::E; ++q) st_cs(dst + ((size_t)(G::TP * q) << p.lg_other), SW ? swap_ri(r.v[q]) : r.v[q]);
                } else if constexpr (DIRECT_OUT) {
                    // natural-order results -> the tile-major ring: the dense tile [row][f] is the memory layout, consecutive
                    // threads = consecutive f then consecutive rows, i.e. every warp instruction writes 256 contiguous bytes
                    const Where w = where(p, bid);
                    cx<T>* dst = p.out + ((uint64_t)zout(p, w.b) << p.lgN) + (size_t)(w.c0 / G::F) * TILE_ELEMS + (size_t)j * G::F + f;
                    B2_UNROLL
                    for (int q = 0; q < G::E; ++q) dst[(size_t)G::TP * q * G::F] = r.v[q];  // write-back stores: pass B re-reads them from L2
                } else {
                    // natural-order results -> dense output tile (the barrier before this phase ended all reads of buf)
                    cx<T>* dst = buf + (size_t)j * G::F + f;
                    B2_UNROLL
                    for (int q = 0; q < G::E; ++q) dst[(size_t)G::TP * q * G::F] = (ROLE == 1 && SW) ? swap_ri(r.v[q]) : r.v[q];
#if defined(__CUDA_ARCH__)
                    tma::fence_proxy_async();  // generic-proxy writes -> visible to the TMA store below
#endif
                }
            }
        } else {
            if (tid == 0 && !DIRECT_OUT) {
                const Where w = where(p, bid);
#if defined(__CUDA_ARCH__)
                issue_store(p, bid, buf);
                tma::bulk_commit();
                tma::bulk_wait_read0();  // shared memory must outlive the store's reads
#else
                cx<T>* dst = p.out + ((uint64_t)zout(p, w.b) << p.lgN) + w.c0;
                for (int e = 0; e < G::L; ++e)
                    for (int f = 0; f < G::F; ++f) dst[((uint64_t)e << p.lg_other) + f] = buf[e * G::F + f];
#endif
            }
        }
    }
};

// ------------------------------------------------------------------------------------------
// Single-launch dataflow four-step.
//
// One persistent grid (one CTA per resident slot) executes BOTH passes of every transform of a batch.
// Work is a single ordered list of tickets handed out by an atomic counter: round r holds the TA tiles of
// pass A of transform r and the TB tiles of pass B of transform r - D, interleaved, so at any moment the
// device is reading new input from HBM (A tiles) and writing finished output to HBM (B tiles) while the
// intermediate lives in a ring of W = 2 D N-element slots that never leaves L2.
//   B(t) may start when all TA tiles of A(t) have been stored     (ready[slot] >= (gen + 1) * TA)
//   A(t) may start when all TB tiles of B(t - W) have been read   (freed[slot] >= gen * TB)
// with slot = t mod W, gen = t / W; both counters only grow.  A dependency always points to a SMALLER ticket,
// and a CTA owns a ticket only while it runs, so the smallest unfinished ticket can always proceed: no
// deadlock whatever the number of co-resident CTAs.  Compared with one launch pair per L2 chunk (the path
// it replaces, ~1000 launches per exec at N = 2^20) there are no per-launch ramps and tails, no host-side
// chunk loop, and reads and writes of HBM are mixed at tile granularity instead of per launch.
// ------------------------------------------------------------------------------------------
struct FlowSched {
    uint32_t batch, TA, TB, D, ring_w, per_round, m, a_big, n_rounds, total;
    B2_HD void decode(uint32_t ticket, int& kind, uint32_t& t, uint32_t& tile, bool& valid) const {
        const uint32_t r = ticket / per_round, i = ticket - r * per_round;
        const uint32_t period = m + 1, k = i / period, j = i - k * period;
        const bool big = j < m;
        tile = big ? k * m + j : k;
        if (big == (a_big != 0)) {
            kind = 0;
            t = r;
            valid = r < batch;
        } else {
            kind = 1;
            t = r - D;
            valid = r >= D && t < batch;
        }
    }
};
// returns false when the ticket count would overflow 32 bits (the caller falls back to the chunked path)
inline bool make_flow_sched(FlowSched& s, uint64_t batch, uint32_t TA, uint32_t TB, uint32_t W) {
    s.TA = TA;
    s.TB = TB;
    s.ring_w = W;
    uint32_t D = W > 2 ? W / 2 : 1;
    if ((uint64_t)D > batch) D = (uint32_t)batch;
    if (D < 1) D = 1;
    s.D = D;
    s.per_round = TA + TB;
    s.a_big = TA >= TB ? 1u : 0u;
    s.m = s.a_big ? TA / TB : TB / TA;
    const uint64_t rounds = batch + D, total = rounds * s.per_round;
    if (batch >= (1ull << 31) || total >= (1ull << 31)) return false;
    s.batch = (uint32_t)batch;
    s.n_rounds = (uint32_t)rounds;
    s.total = (uint32_t)total;
    return true;
}
// control block at the head of the workspace (zeroed before every launch): [0] ticket, [1] error flag,
// [32 .. 32+W) ready counters, [32+W .. 32+2W) freed counters
static constexpr uint32_t FLOW_CTL_HEAD = 32;
inline uint64_t flow_ctl_bytes(uint32_t W) { return ((uint64_t)(FLOW_CTL_HEAD + 2 * W) * 4 + 255) / 256 * 256; }

template <class KA, class KB>
struct FlowKernel {
    using T = typename KA::T;
    static constexpr int NT = KA::NT > KB::NT ? KA::NT : KB::NT;
    static constexpr int MIN_BLOCKS = KA::MIN_BLOCKS < KB::MIN_BLOCKS ? KA::MIN_BLOCKS : KB::MIN_BLOCKS;
    static constexpr size_t SMEM_BYTES = KA::SMEM_BYTES > KB::SMEM_BYTES ? KA::SMEM_BYTES : KB::SMEM_BYTES;
    struct Params {
        typename KA::Params a;
        typename KB::Params b;
        FlowSched sched;
        uint32_t* ctl;
        unsigned long long* trace;  // (B2_FLOW_TRACE builds) per-CTA time stamps, else unused
    };
};

// ------------------------------------------------------------------------------------------
// Device entry point shared by all kernels.
// ------------------------------------------------------------------------------------------
template <class KT, int P>
struct PhaseRunner {
    template <class Regs, class S>
    static B2_HD void run(const typename KT::Params& p, uint32_t bid, int tid, Regs& r, S* smem) {
        KT::template phase<P>(p, bid, tid, r, smem);
#if defined(__CUDA_ARCH__)
        if (P + 1 < KT::NPHASE) __syncthreads();
#endif
        if constexpr (P + 1 < KT::NPHASE) PhaseRunner<KT, P + 1>::run(p, bid, tid, r, smem);
    }
};

#if defined(__CUDACC__)
// minimum CTAs per SM the register allocator must leave room for: 512-thread CTAs would otherwise take
// > 64 registers and run alone on an SM (measured round 1: 1 CTA/SM, 25 % occupancy on the 1024-point tiles)

template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_kernel(const __grid_constant__ typename KT::Params p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename KT::Regs r;
    PhaseRunner<KT, 0>::run(p, blockIdx.x, (int)threadIdx.x, r, reinterpret_cast<cx<typename KT::T>*>(smem_raw));
}

// persistent form of run_kernel (opt-in, B200FFT_PERSIST=1, one-CTA-per-SM geometries such as Direct{16384}): a resident
// CTA walks over tiles bid, bid + gridDim.x, ...; the stores of one tile are still draining while the loads of the next
// are already in flight, and no CTA launch sits between two tiles.  Queued for a timed A/B (not the default).
template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_kernel_persistent(const __grid_constant__ typename KT::Params p, uint32_t n_tiles) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    for (uint32_t bid = blockIdx.x; bid < n_tiles; bid += gridDim.x) {
        typename KT::Regs r;
        PhaseRunner<KT, 0>::run(p, bid, (int)threadIdx.x, r, reinterpret_cast<cx<typename KT::T>*>(smem_raw));
        __syncthreads();  // shared memory is reused by the next tile
    }
}

// same, for kernels whose shared-memory size is run-time data (SmoothKernel)
template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_kernel_dyn(const __grid_constant__ typename KT::Params p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename KT::Regs r;
    PhaseRunner<KT, 0>::run(p, blockIdx.x, (int)threadIdx.x, r, reinterpret_cast<cx<typename KT::T_>*>(smem_raw));
}

// kernels whose steps are run-time data (SmoothConvKernel): step(p, bid, tid, st, smem) for st = 0 .. n_steps - 1 with a
// CTA barrier in between
template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_kernel_loop(const __grid_constant__ typename KT::Params p, uint32_t n_steps) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cx<typename KT::T_>* smem = reinterpret_cast<cx<typename KT::T_>*>(smem_raw);
    for (uint32_t st = 0; st < n_steps; ++st) {
        KT::step(p, blockIdx.x, (int)threadIdx.x, st, smem);
        if (st + 1 < n_steps) __syncthreads();
    }
}

// Thread 0's bookkeeping next to the tiles (all of it off the tiles' critical path):
//   pend   pass-A tile finished earlier by this CTA whose "ready" count has not been published yet.  Publishing
//          needs a device-scope fence that waits for the tile's stores to reach L2; it is DEFERRED to the end of
//          phase 0 of the next tile (by then the stores have long landed, so the fence costs its base latency
//          only and no warp idles on it), or earlier if this CTA is about to block on a dependency.
//   freed  pass-B tile: its ring slot may be overwritten once every thread holds its inputs in registers, i.e.
//          right after the barrier that ends phase 0 (no fence: nothing was written).
//   next   the NEXT ticket is drawn after phase 0 of the current tile and its dependency counter is read after
//          phase 1, so both round trips to L2 overlap the rest of the tile -- but a CTA never holds more than one
//          ticket beyond the one it runs for longer than half a tile: tickets claimed and not yet started are tiles
//          other CTAs may be waiting for (measured with B2_FLOW_TRACE: drawing two tickets ahead made 70 % of the
//          tiles wait ~4 us on their dependency).
struct FlowDep {
    const uint32_t* ptr;  // nullptr: nothing to wait for
    uint32_t target;
};
struct FlowHook {
    uint32_t* pend;
    uint32_t* freed;
    uint32_t* ctl;
    const FlowSched* sc;
    uint32_t next;     // ticket of the next tile
    FlowDep dep;       // its dependency ...
    uint32_t dep_val;  // ... and the counter value seen when it was prefetched
#if defined(B2_FLOW_TRACE)
    unsigned long long* trace;  // thread 0 of the first CTAs: globaltimer stamps at the phase boundaries of every tile
    uint32_t n;
#endif
};
#if defined(B2_FLOW_TRACE)
static constexpr uint32_t FLOW_TRACE_CTAS = 32, FLOW_TRACE_WORDS = 4096;
B2_D void flow_stamp(FlowHook& h, int tid, unsigned long long tag) {
    if (tid == 0 && h.trace && h.n + 1 < FLOW_TRACE_WORDS) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        h.trace[h.n++] = (t << 8) | tag;
    }
}
#define B2_STAMP(h, tid, tag) flow_stamp(h, tid, tag)
#else
#define B2_STAMP(h, tid, tag)
#endif
B2_D void flow_publish(uint32_t*& pend) {
    if (pend) {
        __threadfence();
        atomicAdd(pend, 1u);
        pend = nullptr;
    }
}
B2_D uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// spin until *ctr >= target (bounded: a scheduling bug raises the error flag instead of hanging the GPU)
B2_D void flow_spin(uint32_t* ctl, const uint32_t* ctr, uint32_t target) {
    uint32_t spins = 0;
    while (ld_relaxed_u32(ctr) < target) {
        __nanosleep(spins < 64 ? 32 : 256);
        if (++spins > (1u << 22) || (spins > 4096 && ld_relaxed_u32(ctl + 1) != 0)) {
            atomicExch(ctl + 1, 1u);
            break;
        }
    }
}
B2_D FlowDep flow_dep(const FlowSched& sc, const uint32_t* ctl, uint32_t ticket) {
    FlowDep d{nullptr, 0u};
    if (ticket >= sc.total) return d;
    int kind;
    uint32_t t, tile;
    bool valid;
    sc.decode(ticket, kind, t, tile, valid);
    if (!valid) return d;
    const uint32_t* ready = ctl + FLOW_CTL_HEAD;
    const uint32_t* freed = ready + sc.ring_w;
    const uint32_t gen = t / sc.ring_w, slot = t - gen * sc.ring_w;
    if (kind == 0) {
        if (gen > 0) {
            d.ptr = freed + slot;
            d.target = gen * sc.TB;
        }
    } else {
        d.ptr = ready + slot;
        d.target = (gen + 1u) * sc.TA;
    }
    return d;
}
B2_D void flow_draw_next(FlowHook& h) { h.next = atomicAdd(h.ctl, 1u); }
B2_D void flow_peek_dep(FlowHook& h) {
    h.dep = flow_dep(*h.sc, h.ctl, h.next);
    h.dep_val = h.dep.ptr ? ld_relaxed_u32(h.dep.ptr) : 0u;
}
// phases of one tile inside a CTA that may have more threads than the tile's kernel uses
template <class KT, int NTC, int P>
struct FlowPhases {
    static_assert(KT::NPHASE >= 3, "dataflow tiles have at least two stages");
    static B2_D void run(const typename KT::Params& p, uint32_t bid, int tid, typename KT::Regs& r, cx<typename KT::T>* smem,
                         FlowHook& hook) {
        if (NTC == KT::NT || tid < KT::NT) KT::template phase<P>(p, bid, tid, r, smem);
        B2_STAMP(hook, tid, 0x10 + 2 * P);  // thread 0 finished phase P
        if constexpr (P == 0) {
            if (tid == 0) flow_publish(hook.pend);
        }
        if constexpr (P + 1 < KT::NPHASE) {
            __syncthreads();
            B2_STAMP(hook, tid, 0x11 + 2 * P);  // everybody finished phase P
            if constexpr (P == 0) {
                if (tid == 0) {
                    if (hook.freed) atomicAdd(hook.freed, 1u);
                    flow_draw_next(hook);
                }
            }
            if constexpr (P == 1) {
                if (tid == 0) flow_peek_dep(hook);
            }
            FlowPhases<KT, NTC, P + 1>::run(p, bid, tid, r, smem, hook);
        }
    }
};

template <class KA, class KB>
__global__ void __launch_bounds__(FlowKernel<KA, KB>::NT, FlowKernel<KA, KB>::MIN_BLOCKS)
run_flow(const __grid_constant__ typename FlowKernel<KA, KB>::Params p) {
    using FK = FlowKernel<KA, KB>;
    using C = cx<typename FK::T>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ uint32_t s_next[2];
    C* smem = reinterpret_cast<C*>(smem_raw);
    const int tid = (int)threadIdx.x;
    const FlowSched& sc = p.sched;
    uint32_t* ready = p.ctl + FLOW_CTL_HEAD;
    uint32_t* freed = ready + sc.ring_w;
    FlowHook hook;
    hook.pend = nullptr;
    hook.freed = nullptr;
    hook.ctl = p.ctl;
    hook.sc = &sc;
    hook.next = 0;
    hook.dep = FlowDep{nullptr, 0u};
    hook.dep_val = 0;
#if defined(B2_FLOW_TRACE)
    hook.trace = (p.trace && blockIdx.x < FLOW_TRACE_CTAS) ? p.trace + (size_t)blockIdx.x * FLOW_TRACE_WORDS : nullptr;
    hook.n = 0;
#endif
    if (tid == 0) {
        flow_draw_next(hook);
        flow_peek_dep(hook);
        if (hook.dep.ptr && hook.dep_val < hook.dep.target) flow_spin(p.ctl, hook.dep.ptr, hook.dep.target);
        s_next[0] = hook.next;
    }
    __syncthreads();
    for (uint32_t it = 0;; ++it) {
        const uint32_t ticket = s_next[it & 1u];
        if (ticket >= sc.total) break;
        int kind;
        uint32_t t, tile;
        bool valid;
        sc.decode(ticket, kind, t, tile, valid);
        B2_STAMP(hook, tid, valid ? (kind == 0 ? 0x01 : 0x02) : 0x03);  // tile start
        if (valid) {
            const uint32_t slot = t % sc.ring_w;
            if (kind == 0) {
                typename KA::Regs r;
                hook.freed = nullptr;
                FlowPhases<KA, FK::NT, 0>::run(p.a, t * sc.TA + tile, tid, r, smem, hook);
                hook.pend = ready + slot;  // published later (see FlowHook)
            } else {
                typename KB::Regs r;
                hook.freed = freed + slot;
                FlowPhases<KB, FK::NT, 0>::run(p.b, t * sc.TB + tile, tid, r, smem, hook);
            }
        } else if (tid == 0) {  // empty ticket (first / last rounds): nothing to overlap with
            flow_draw_next(hook);
            flow_peek_dep(hook);
        }
        B2_STAMP(hook, tid, 0x04);  // tile body done (thread 0)
        if (tid == 0) {
            if (hook.dep.ptr && hook.dep_val < hook.dep.target) {
                flow_publish(hook.pend);  // never block while other tiles may be waiting for ours
                flow_spin(p.ctl, hook.dep.ptr, hook.dep.target);
                B2_STAMP(hook, tid, 0x05);  // had to wait for the next tile's dependency
            }
            s_next[(it + 1u) & 1u] = hook.next;
        }
        __syncthreads();  // shared memory is reused by the next tile; mailbox visible
    }
    if (tid == 0) flow_publish(hook.pend);
#if defined(B2_FLOW_TRACE)
    if (tid == 0 && hook.trace) hook.trace[FLOW_TRACE_WORDS - 1] = hook.n;
#endif
}

// TMA-tiled passes: one thread starts the tile's load, everybody waits on the mbarrier it completes on
template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_kernel_tma(const __grid_constant__ typename KT::Params p) {
    // no static shared memory in this kernel: the dynamic window then starts at offset 0 of the CTA's shared memory,
    // which gives the tile the 128-byte alignment tensor copies need; the mbarrier sits behind the tile
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using T = typename KT::T;
    unsigned char* base = smem_raw + ((128u - (tma::smem_u32(smem_raw) & 127u)) & 127u);  // (the launch reserves the slack)
    cx<T>* buf = reinterpret_cast<cx<T>*>(base);
    uint64_t* bar = reinterpret_cast<uint64_t*>(base + KT::SMEM_BYTES);
    const int tid = (int)threadIdx.x;
    if (tid == 0) {
        tma::mbar_init(bar, 1);
        tma::fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) KT::issue_load(p, blockIdx.x, buf, bar);
    typename KT::Regs r;
    KT::prefetch(p, blockIdx.x, tid, r);  // table loads overlap the tile's flight
    tma::mbar_wait(bar, 0);
    PhaseRunner<KT, 0>::run(p, blockIdx.x, tid, r, buf);
}

template <class KT>
__global__ void __launch_bounds__(KT::NT, KT::MIN_BLOCKS) run_pipelined(const __grid_constant__ typename KT::Params p) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    using T = typename KT::T;
    cx<T>* buf0 = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* buf1 = reinterpret_cast<cx<T>*>(smem_raw + KT::BUF_BYTES);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + 2 * KT::BUF_BYTES);
    const int tid = (int)threadIdx.x;
    if (tid == 0) {
        tma::mbar_init(&bar[0], 1);
        tma::mbar_init(&bar[1], 1);
        tma::fence_mbar_init();
    }
    __syncthreads();
    uint32_t item = blockIdx.x;
    if (tid == 0 && item < p.n_items) {
        const uint32_t bytes = KT::fetch_bytes(p, item);
        tma::mbar_arrive_expect_tx(&bar[0], bytes);
        tma::bulk_g2s(buf0, KT::fetch_src(p, item), bytes, &bar[0]);
    }
    for (uint32_t it = 0; item < p.n_items; item += gridDim.x, ++it) {
        const uint32_t cur = it & 1u;
        cx<T>* buf = cur ? buf1 : buf0;
        const uint32_t next = item + gridDim.x;
        if (tid == 0 && next < p.n_items) {
            // the other buffer was last touched (generic proxy) before the final barrier of the previous tile
            tma::fence_proxy_async();
            const uint32_t bytes = KT::fetch_bytes(p, next);
            tma::mbar_arrive_expect_tx(&bar[cur ^ 1u], bytes);
            tma::bulk_g2s(cur ? buf0 : buf1, KT::fetch_src(p, next), bytes, &bar[cur ^ 1u]);
        }
        tma::mbar_wait(&bar[cur], (it >> 1) & 1u);
        typename KT::Regs r;
        PhaseRunner<KT, 0>::run(p, item, tid, r, buf);
    }
}
#endif

}  // namespace b2
