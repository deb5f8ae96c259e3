// b200fft -- common definitions shared by the sm_90a kernels and the host planner.
//
// Every kernel body in this library is written as a sequence of `phase<P>()` functions that are
// separated by a CTA-wide barrier.  On the GPU `run_kernel<K>` calls them back to back with
// __syncthreads() in between; the test-only CPU harness (tests/emu) replays the same phases
// thread by thread so that index maths, twiddle tables and planning can be checked without a GPU.
#pragma once

#include <cstddef>
#include <cstdint>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#define B2_D __device__ __forceinline__
#else
#define B2_HD inline
#define B2_D inline
#endif

#if defined(__CUDA_ARCH__)
#define B2_UNROLL _Pragma("unroll")
#else
#define B2_UNROLL
#endif

// Twiddle loads: by default a radix-R stage loads only W^(k 2^i) (log2 R table entries) and builds the other
// R-1-log2 R factors as products, and the inter-pass twiddles of a four-step row come from 1 + log2 E table entries
// per thread instead of E: every table load removed is an LSU request removed, for a relative L2 error
// +5 % (tests/test_emu_parity.py).  -DB2_TW_ALL restores one table load per factor.
#if !defined(B2_TW_ALL)
#if !defined(B2_TW_FEW)
#define B2_TW_FEW 1
#endif
#if !defined(B2_TWROW_FEW)
#define B2_TWROW_FEW 1
#endif
#endif

namespace b2 {

// Complex<T> of the reference is repr(C) {re, im} (CHANGELOG.md:139) == float2 / double2.
template <typename T>
struct alignas(2 * sizeof(T)) cx {
    T x, y;
};

template <typename T> B2_HD cx<T> mk(T x, T y) { cx<T> r; r.x = x; r.y = y; return r; }

// ---- complex arithmetic ------------------------------------------------------------------------
// Hopper has no packed FP32 instructions, so complex<f32> arithmetic is scalar FADD / FMUL / FFMA.  On the
// device the complex products are written as explicit FMAs, cmul = (fma(-a.y, w.y, a.x*w.x), fma(a.x, w.y,
// a.y*w.x)), so that their rounding is fixed by the source rather than by the compiler's contraction choice.
template <typename T> B2_HD cx<T> operator+(cx<T> a, cx<T> b) { return mk<T>(a.x + b.x, a.y + b.y); }
template <typename T> B2_HD cx<T> operator-(cx<T> a, cx<T> b) { return mk<T>(a.x - b.x, a.y - b.y); }
// (a.x + i a.y)(w.x + i w.y)
template <typename T> B2_HD cx<T> cmul(cx<T> a, cx<T> w) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(-a.y, w.y, __fmul_rn(a.x, w.x)), __fmaf_rn(a.x, w.y, __fmul_rn(a.y, w.x)));
#endif
    return mk<T>(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x);
}
// a * conj(w)
template <typename T> B2_HD cx<T> cmulc(cx<T> a, cx<T> w) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(a.y, w.y, __fmul_rn(a.x, w.x)), __fmaf_rn(-a.x, w.y, __fmul_rn(a.y, w.x)));
#endif
    return mk<T>(a.x * w.x + a.y * w.y, a.y * w.x - a.x * w.y);
}
// a * s (real scalar)
template <typename T> B2_HD cx<T> scale(cx<T> a, T s) { return mk<T>(a.x * s, a.y * s); }
// a + s * b, s real
template <typename T> B2_HD cx<T> axpy(cx<T> a, T s, cx<T> b) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) return mk<T>(__fmaf_rn(b.x, s, a.x), __fmaf_rn(b.y, s, a.y));
#endif
    return mk<T>(a.x + s * b.x, a.y + s * b.y);
}
template <typename T> B2_HD cx<T> conj(cx<T> a) { return mk<T>(a.x, -a.y); }
// multiply by -i  (forward quarter turn, twiddle(1,4))
template <typename T> B2_HD cx<T> mul_mi(cx<T> a) { return mk<T>(a.y, -a.x); }
// a + (-i) b   and   a - (-i) b : the quarter turn rides on the add's operand modifiers
template <typename T> B2_HD cx<T> add_mi(cx<T> a, cx<T> b) { return mk<T>(a.x + b.y, a.y - b.x); }
template <typename T> B2_HD cx<T> sub_mi(cx<T> a, cx<T> b) { return mk<T>(a.x - b.y, a.y + b.x); }
// swap re <-> im.  ifft(x) = swap(fft(swap(x))): the whole inverse direction is a register
// renaming at the outermost load and store of a plan, every table stays "forward".
template <typename T> B2_HD cx<T> swap_ri(cx<T> a) { return mk<T>(a.y, a.x); }

// Table loads (stage twiddles, chirps, multipliers): read-only path, kept in L1 with evict-last priority.
// With plain __ldg/__ldcs the streaming signal traffic evicts the few KiB of twiddles every tile, and most
// twiddle loads go to L2.
template <typename T> B2_HD cx<T> ldg(const cx<T>* p) {
#if defined(__CUDA_ARCH__)
    cx<T> r;
    if constexpr (sizeof(T) == 4) {
        asm("ld.global.nc.L1::evict_last.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
    } else {
        asm("ld.global.nc.L1::evict_last.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
    }
    return r;
#else
    return *p;
#endif
}
// bring the line holding *p into L1 ahead of an ldg of it (no register is held while the line is in flight)
template <typename T> B2_HD void prefetch_l1(const T* p) {
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}
// large read-only tables that are streamed once per CTA (the N-entry inter-pass twiddle table): L2 only
template <typename T> B2_HD cx<T> ldg_stream(const cx<T>* p) {
#if defined(__CUDA_ARCH__)
    cx<T> r;
    if constexpr (sizeof(T) == 4) {
        asm("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
    } else {
        asm("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
    }
    return r;
#else
    return *p;
#endif
}
B2_HD uint32_t ldg_u32(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// Signal data is read once and written once: no L1 allocation, and an L2 evict-first policy so that dead
// lines (consumed input, finished output, the already-read half of the workspace) leave L2 before the
// lines still waiting to be used.  The workspace written by a first pass gets the opposite hint
// (evict-last) until the second pass has read it.
#if defined(__CUDACC__)
B2_D unsigned long long l2_evict_first() {
    unsigned long long p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
B2_D unsigned long long l2_evict_last() {
    unsigned long long p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
#endif
template <typename T> B2_HD cx<T> ld_stream(const cx<T>* p) {
#if defined(__CUDA_ARCH__)
    cx<T> r;
    if constexpr (sizeof(T) == 4) {
        asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;"
                     : "=f"(r.x), "=f"(r.y) : "l"(p), "l"(l2_evict_first()));
    } else {
        asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;"
                     : "=d"(r.x), "=d"(r.y) : "l"(p), "l"(l2_evict_first()));
    }
    return r;
#else
    return *p;
#endif
}
template <typename T> B2_HD void st_stream(cx<T>* p, cx<T> v) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y),
                     "l"(l2_evict_first()) : "memory");
    } else {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y),
                     "l"(l2_evict_first()) : "memory");
    }
#else
    *p = v;
#endif
}
// scalar forms of ld_stream / st_stream for real rows
template <typename T> B2_HD T ld_stream_r(const T* p) {
#if defined(__CUDA_ARCH__)
    T r;
    if constexpr (sizeof(T) == 4) {
        asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(l2_evict_first()));
    } else {
        asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(r) : "l"(p), "l"(l2_evict_first()));
    }
    return r;
#else
    return *p;
#endif
}
template <typename T> B2_HD void st_stream_r(T* p, T v) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(l2_evict_first()) : "memory");
    } else {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(l2_evict_first()) : "memory");
    }
#else
    *p = v;
#endif
}

// "cache streaming" forms (ld/st.global.cs): what the four-step passes use.  Chosen by A/B timing:
// the explicit no-allocate + L2-hint forms above are better for the one-pass Direct kernels, the .cs forms
// for the two L2-coupled passes.
template <typename T> B2_HD cx<T> ld_cs(const cx<T>* p) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) {
        float2 v = __ldcs(reinterpret_cast<const float2*>(p));
        return mk<T>(v.x, v.y);
    } else {
        double2 v = __ldcs(reinterpret_cast<const double2*>(p));
        return mk<T>(v.x, v.y);
    }
#else
    return *p;
#endif
}
template <typename T> B2_HD void st_cs(cx<T>* p, cx<T> v) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) {
        __stcs(reinterpret_cast<float2*>(p), make_float2(v.x, v.y));
    } else {
        __stcs(reinterpret_cast<double2*>(p), make_double2(v.x, v.y));
    }
#else
    *p = v;
#endif
}
// strong relaxed load at device scope (SASS LDG.E.64.STRONG.GPU): never served from this SM's L1, so data written
// by other SMs earlier in the SAME launch (the dataflow four-step's ring) is read from L2, the point of coherence
template <typename T> B2_HD cx<T> ld_strong(const cx<T>* p) {
#if defined(__CUDA_ARCH__)
    cx<T> r;
    if constexpr (sizeof(T) == 4) {
        asm volatile("ld.relaxed.gpu.global.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p) : "memory");
    } else {
        asm volatile("ld.relaxed.gpu.global.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p) : "memory");
    }
    return r;
#else
    return *p;
#endif
}
// drop a 128-byte line of dead scratch data from L2 WITHOUT writing it back (PTX discard.global.L2).  Used on the
// two-pass intermediate right after the second pass has it in registers: without it, much of the
// intermediate is written back to HBM when its dirty lines are evicted.
B2_HD void l2_discard_line(const void* p128) {
#if defined(__CUDA_ARCH__)
    asm volatile("discard.global.L2 [%0], 128;" ::"l"(p128) : "memory");
#else
    (void)p128;
#endif
}
// store into the L2-resident workspace that the next pass re-reads
template <typename T> B2_HD void st_keep(cx<T>* p, cx<T> v) {
#if defined(__CUDA_ARCH__)
    if constexpr (sizeof(T) == 4) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y),
                     "l"(l2_evict_last()) : "memory");
    } else {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y),
                     "l"(l2_evict_last()) : "memory");
    }
#else
    *p = v;
#endif
}

// opaque 128-byte tensor-map descriptor (CUtensorMap of the driver API; built on the host by rt::make_tile_map,
// consumed by cp.async.bulk.tensor in tma.h).  The CPU replay harness never reads it.
struct alignas(64) TMap {
    unsigned long long opaque[16];
};

// compile-time list of stage radices
template <int... Rs>
struct Radices {
    static constexpr int N = sizeof...(Rs);
    static constexpr int get(int i) {
        constexpr int a[] = {Rs...};
        return a[i];
    }
    static constexpr int product(int upto = N) {  // product of the first `upto` radices
        constexpr int a[] = {Rs...};
        int p = 1;
        for (int i = 0; i < upto; ++i) p *= a[i];
        return p;
    }
    // offset (in elements) of stage s inside the packed stage-twiddle table; stage 0 has none
    static constexpr int tw_offset(int s) {
        constexpr int a[] = {Rs...};
        int off = 0, p = 1;
        for (int i = 0; i < s; ++i) {
            if (i >= 1) off += (a[i] - 1) * p;
            p *= a[i];
        }
        return off;
    }
    static constexpr int tw_total() { return tw_offset(N); }
    static constexpr bool all_pow2() {
        constexpr int a[] = {Rs...};
        for (int i = 0; i < N; ++i)
            if (a[i] & (a[i] - 1)) return false;
        return true;
    }
};

template <int A, int B> struct StaticMax { static constexpr int v = A > B ? A : B; };

}  // namespace b2
