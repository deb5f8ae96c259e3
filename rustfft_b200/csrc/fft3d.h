// Compiled power-of-two FFT pass down a strided axis (the H and D axes of the 3-D plans, impl.inl): data viewed as
// [outer][N][inner], column g = o * inner + c holds element n at o * N * inner + n * inner + c.
//
//   AxisKernel<G, SW> = FftKernel<G, FF, FF, LoadAxis<T, SW>, StoreAxis<T, SW>>   one CTA: F adjacent columns, N = G::L points each
//
// Consecutive threads take consecutive columns (the engine's "f fastest" mapping on both sides), so one row of a tile is a run of
// F * sizeof(cx<T>) bytes.  A tile may span two slabs (inner < F, or inner not a multiple of F); only a launch's last CTA masks
// columns.  Every thread holds its whole share of the tile in registers before the first store (FftKernel's phase 0 loads, the
// last phase stores, with CTA barriers between), so the pass runs in place as well as out of place.  Loads and stores are one-pass
// streaming accesses: each element is read once and written once per pass.  An inverse plan swaps re / im on the load and on the
// store (ifft(x) = swap(fft(swap(x))), common.h).
#pragma once
#include "kernels.h"

namespace b2 {

// g -> (o, c): o = g / cols, c = g - o * cols, with `cols` the columns per slab in this launch's view (the slab's width, or, for a
// launch over one column range of a slab wider than 2^30 columns, any divisor larger than the launch).  g < 2^31 (FastDiv).
template <typename T, bool SWAP>
struct LoadAxis {
    const cx<T>* in;   // column 0 of the launch
    uint64_t slab;     // N * inner elements
    uint32_t stride;   // inner: elements between n and n + 1
    FastDiv cols;
    struct St { const cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t o = cols.div((uint32_t)g), c = (uint32_t)g - o * cols.d;
        return St{in + o * slab + c, ok};
    }
    B2_HD cx<T> get(const St& s, int e) const {
        if (!s.ok) return mk<T>(0, 0);
        cx<T> v = ld_stream(s.p + (size_t)e * stride);
        return SWAP ? swap_ri(v) : v;
    }
};

template <typename T, bool SWAP>
struct StoreAxis {
    cx<T>* out;
    uint64_t slab;
    uint32_t stride;
    FastDiv cols;
    struct St { cx<T>* p; bool ok; };
    B2_HD St prep(uint64_t g, bool ok) const {
        const uint32_t o = cols.div((uint32_t)g), c = (uint32_t)g - o * cols.d;
        return St{out + o * slab + c, ok};
    }
    B2_HD void put(const St& s, int e, cx<T> v) const {
        if (s.ok) st_stream(s.p + (size_t)e * stride, SWAP ? swap_ri(v) : v);
    }
};

// resident CTAs per SM the register allocator plans for: the engine's default, except that 512-thread CTAs of 16 f64 elements per
// thread (32 data registers of 64 bits) get the whole register file (their tile of 139 KiB allows one CTA per SM anyway)
constexpr int axis_min_blocks(int nt, int e, int esz) { return (esz == 16 && e >= 16) ? 1 : default_min_blocks(nt, e); }

template <class G, bool SW>
struct AxisKernel : FftKernel<G, FF, FF, LoadAxis<typename G::T, SW>, StoreAxis<typename G::T, SW>> {
    static constexpr int MIN_BLOCKS = axis_min_blocks(G::NT, G::E, (int)sizeof(cx<typename G::T>));
};

}  // namespace b2
