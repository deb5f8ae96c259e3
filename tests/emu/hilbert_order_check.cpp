// TEST INFRASTRUCTURE -- NOT PRODUCT CODE (tests/test_hilbert.py::test_fused_kernel_is_thread_order_independent builds and runs it).
// Thread-order race check of HilbertKernel<G> on the CPU: every phase runs its NT threads once in order and once in reverse (and
// once in a shuffled order); a shared-memory race inside a phase (one thread reading or writing a slot another thread writes
// between the same two barriers) makes the results depend on the order.  Shared memory is poisoned (NaN) before each run.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
#include "../../rustfft_b200/csrc/common.h"
#include "../../rustfft_b200/csrc/hilbert.h"
using namespace b2;

template <class KT, int P>
struct Run {
    static void go(const typename KT::Params& p, uint32_t bid, std::vector<typename KT::Regs>& regs, cx<typename KT::T>* smem,
                   const std::vector<int>& order) {
        for (int tid : order) KT::template phase<P>(p, bid, tid, regs[(size_t)tid], smem);
        if constexpr (P + 1 < KT::NPHASE) Run<KT, P + 1>::go(p, bid, regs, smem, order);
    }
};

template <class G>
int check(const char* name, uint32_t rows) {
    using KT = HilbertKernel<G>;
    using T = typename G::T;
    const int M = G::L;
    std::mt19937 rng(M);
    std::normal_distribution<double> nd;
    std::vector<T> x((size_t)rows * 2 * M);
    for (auto& v : x) v = (T)nd(rng);
    std::vector<cx<T>> tab(M), tw(std::max(1, G::TW_ELEMS));
    for (auto& v : tab) v = mk<T>((T)nd(rng), (T)nd(rng));
    for (auto& v : tw) v = mk<T>((T)nd(rng), (T)nd(rng));
    const uint32_t ctas = (rows + G::F - 1) / G::F;
    std::vector<std::vector<cx<T>>> outs;
    for (int variant = 0; variant < 3; ++variant) {
        std::vector<int> order(KT::NT);
        for (int i = 0; i < KT::NT; ++i) order[i] = i;
        if (variant == 1) std::reverse(order.begin(), order.end());
        if (variant == 2) std::shuffle(order.begin(), order.end(), rng);
        std::vector<cx<T>> out((size_t)rows * 2 * M, mk<T>(-7, -7));
        typename KT::Params p{};
        p.in = x.data();
        p.out = out.data();
        p.tab = tab.data();
        p.tw = tw.data();
        p.rows = rows;
        std::vector<typename KT::Regs> regs((size_t)KT::NT);
        std::vector<cx<T>> smem(KT::SMEM_BYTES / sizeof(cx<T>) + 1);
        for (uint32_t bid = 0; bid < ctas; ++bid) {
            std::memset(smem.data(), 0xff, smem.size() * sizeof(smem[0]));
            Run<KT, 0>::go(p, bid, regs, smem.data(), order);
        }
        outs.push_back(out);
    }
    const bool same = std::memcmp(outs[0].data(), outs[1].data(), outs[0].size() * sizeof(cx<T>)) == 0 &&
                      std::memcmp(outs[0].data(), outs[2].data(), outs[0].size() * sizeof(cx<T>)) == 0;
    bool finite = true;
    for (auto& v : outs[0]) finite = finite && v.x == v.x && v.y == v.y;
    std::printf("%s %s M=%d F=%d NT=%d rows=%u: %s\n", same && finite ? "ok  " : "FAIL", name, M, G::F, KT::NT, rows,
                same ? (finite ? "order-independent, finite" : "order-independent, NON-FINITE") : "ORDER-DEPENDENT");
    return same && finite ? 0 : 1;
}

// the Direct geometries of impl.inl (B2_DIRECT / B2_DIRECT_V1) the fused path instantiates, smallest to largest
int main() {
    int bad = 0;
    bad += check<Geo<float, 2, 2, 128, Radices<2>>>("f32", 129);
    bad += check<Geo<float, 8, 8, 128, Radices<8>>>("f32", 129);
    bad += check<Geo<float, 16, 4, 32, Radices<4, 4>>>("f32", 33);
    bad += check<Geo<float, 256, 16, 8, Radices<16, 16>>>("f32", 17);
    bad += check<Geo<float, 2048, 16, 2, Radices<8, 16, 16>>>("f32", 3);
    bad += check<Geo<float, 8192, 16, 1, Radices<2, 16, 16, 16>>>("f32", 2);
    bad += check<Geo<float, 16384, 32, 1, Radices<16, 32, 32>>>("f32", 2);
    bad += check<Geo<double, 2, 2, 128, Radices<2>>>("f64", 129);
    bad += check<Geo<double, 8, 8, 64, Radices<8>>>("f64", 65);
    bad += check<Geo<double, 256, 8, 8, Radices<4, 8, 8>>>("f64", 17);
    bad += check<Geo<double, 1024, 8, 2, Radices<2, 8, 8, 8>>>("f64", 3);
    bad += check<Geo<double, 8192, 8, 1, Radices<2, 8, 8, 8, 8>>>("f64", 2);
    std::printf(bad ? "RACE CHECK FAILED\n" : "RACE CHECK OK\n");
    return bad;
}
