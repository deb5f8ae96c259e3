// Chirp-z transforms on the unit circle: the kernels of the general path (L = next_pow2(n + m - 1) > 4096), one per step
// around the library's own L-point plans.  The fused path (L <= 4096) is BluesteinKernel (kernels.h) with CZT tables.
//
//   CztPreKernel    workspace row r, element t < L:  x[r][t] pre[t] for t < n, else 0          (real or complex rows)
//   (the L-point forward plan, in place)
//   CztMulKernel    every workspace element times mult[t mod L]                               (mult = FFT_L(b) / L)
//   (the L-point inverse plan, in place: the circular convolution of x pre with b)
//   CztPostKernel   y[r][k] = post[k] w[r][k] for k < m
//
// Launches cover rows * L (rows * m) elements of one workspace chunk, below 2^31 (the caller's chunks of whole rows).
#pragma once
#include "kernels.h"

namespace b2 {

template <typename TT, bool REAL>
struct CztPreKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const void* in;     // rows of n samples: cx<T>, or T when REAL
        cx<T>* out;         // rows of L
        const cx<T>* pre;   // n entries
        uint64_t n_elem;    // rows * L
        uint32_t n, lg_l;   // row length, log2 L
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t row = (uint32_t)(i >> p.lg_l), t = (uint32_t)i & ((1u << p.lg_l) - 1);
        cx<T> v = mk<T>(0, 0);
        if (t < p.n) {
            const uint64_t s = (uint64_t)row * p.n + t;
            if constexpr (REAL) {
                v.x = ld_stream_r((const T*)p.in + s);
            } else {
                v = ld_stream((const cx<T>*)p.in + s);
            }
            v = cmul(v, ldg(p.pre + t));
        }
        p.out[i] = v;
    }
};

template <typename TT>
struct CztMulKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        cx<T>* w;            // rows of L, in place
        const cx<T>* mult;   // L entries
        uint64_t n_elem;     // rows * L
        uint32_t mask;       // L - 1
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        p.w[i] = cmul(p.w[i], ldg(p.mult + ((uint32_t)i & p.mask)));
    }
};

template <typename TT>
struct CztPostKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const cx<T>* w;      // rows of L
        cx<T>* out;          // rows of m
        const cx<T>* post;   // m entries
        uint64_t n_elem;     // rows * m
        uint32_t lg_l;
        FastDiv div_m;       // by m
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t row = p.div_m.div((uint32_t)i), k = (uint32_t)i - row * p.div_m.d;
        st_stream(p.out + i, cmul(p.w[((uint64_t)row << p.lg_l) + k], ldg(p.post + k)));
    }
};

}  // namespace b2
