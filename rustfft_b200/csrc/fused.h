// Fused single-launch four-step: ONE persistent, warp-specialised kernel runs both passes of every transform of a batch.
//
// Why: the chunked path (one launch pair per L2 chunk, kernels.h run_kernel_tma) is latency bound -- a tile's load, its
// butterflies and its store are strictly serial inside a CTA, an SM holds two such tiles, and every ~10 us launch pays a
// ramp and a tail (low occupancy, DRAM about half busy).  Here every SM runs one
// resident CTA made of
//     1 scheduler thread  draws tile tickets from a global counter, waits for the ticket's dependency (always a
//                         SMALLER ticket) and hands the tile to the producer through a two-entry queue;
//     1 producer thread   queues the tile's TMA load into the next free shared-memory stage;
//     NG consumer groups  (NTG threads each, one tile at a time): wait for the stage's mbarrier, run the tile's FFTs in
//                         registers + in place in the stage buffer (the phases of TmaTileKernel), leave the finished
//                         dense tile in the same buffer;
//     1 storer thread     TMA-stores finished tiles, frees the stage once the store has read it, publishes the
//                         "pass-A tile landed" counters;
// the scheduler, producer and storer warps (plus one idle warp) form one warpgroup that gives up registers with
// setmaxnreg, so that the consumer warpgroups can hold a tile's 32 values per thread without spilling;
// so the load of tile i+2, the butterflies of tiles i and i+1 and the store of tile i-1 overlap inside one SM, there
// are no launches between tiles, and the device mixes HBM reads (pass-A tiles) with HBM writes (pass-B tiles) at tile
// granularity.  Ticket order = FlowSched (kernels.h): round r holds the pass-A tiles of transform r interleaved with
// the pass-B tiles of transform r - D; the intermediate lives in a ring of W = 2 D transform slots that stays in L2
// (pass B drops the lines it has consumed with discard.global.L2, so they are never written back to HBM).
//   B(t) may start when all TA tiles of A(t) have landed    (ready[slot] >= (gen + 1) * TA)
//   A(t) may start when all TB tiles of B(t - W) were read  (freed[slot] >= gen * TB)
// Both counters only grow; a dependency always points to a smaller ticket and a CTA's consumers / storer never wait
// for its producer, so the smallest unfinished ticket can always proceed: no deadlock whatever the co-residency.
// The reference's shape for the same job: MixedRadix's six steps (src/algorithm/mixed_radix.rs:128-158).
#pragma once
#include "kernels.h"

namespace b2 {

template <class KA, class KB, int NG_, int NS_>
struct FusedKernel {
    using T = typename KA::T;
    static constexpr int NG = NG_;      // consumer groups
    static constexpr int NSTAGE = NS_;  // shared-memory stages (tiles in flight per SM)
    static constexpr int NTG = KA::NT;  // threads per consumer group
    static_assert(KA::NT == KB::NT, "both passes use the same consumer-group size");
    static_assert(KA::TILE_BYTES == KB::TILE_BYTES, "both passes move tiles of the same size");
    static_assert(NTG % 32 == 0 && NSTAGE <= 8 && NG <= 8, "geometry");
    // consumer groups first, then ONE service warpgroup (producer, storer, scheduler, spare warp): setmaxnreg acts on whole
    // warpgroups, so the service roles can hand their registers to the consumers only if no consumer warp shares their group
    static_assert(NG * NTG % 128 == 0, "consumer groups fill whole warpgroups");
    static constexpr int NT = NG * NTG + 128;
    static constexpr int SVC_WARP = NG * NTG / 32;  // first warp of the service warpgroup
    // register budgets: the launch grants every thread LAUNCH_REGS (__launch_bounds__(NT, 1) over the 64 K register file,
    // rounded down to the allocation granule of 8); the service warpgroup shrinks to SVC_REGS and the consumers grow to
    // CONS_REGS, claiming no more than the service warpgroup released
    static constexpr int LAUNCH_REGS = 65536 / NT / 8 * 8;
    static constexpr int SVC_REGS = 32;  // 24 spills in the scheduler and producer loops
    static constexpr int CONS_REGS = (LAUNCH_REGS * NT - SVC_REGS * 128) / (NG * NTG) / 8 * 8;
    static_assert(CONS_REGS * NG * NTG + SVC_REGS * 128 <= LAUNCH_REGS * NT && CONS_REGS >= LAUNCH_REGS && CONS_REGS <= 256,
                  "setmaxnreg budgets must not overcommit the registers the launch granted");
    static constexpr int NQ = 2;              // tiles the scheduler may run ahead of the producer
    static constexpr size_t STAGE_BYTES = ((KA::SMEM_BYTES > KB::SMEM_BYTES ? KA::SMEM_BYTES : KB::SMEM_BYTES) + 127) / 128 * 128;
    static constexpr size_t CTRL_BYTES = 512;  // 4 * NSTAGE + 2 * NQ mbarriers, (NSTAGE + NQ) x {kind, tile, slot, -}
    static constexpr size_t SMEM_BYTES = (size_t)NSTAGE * STAGE_BYTES + CTRL_BYTES + 128;  // + alignment slack
    struct Params {
        typename KA::Params a;
        typename KB::Params b;
        FlowSched sched;
        uint32_t* ctl;    // control block (FLOW_CTL_HEAD layout of kernels.h), zeroed before the launch
        unsigned long long* trace;  // B200FFT_FUSED_TRACE=1: %globaltimer stamps of the first CTAs' pipeline events, else null
        uint32_t flags;   // bit 0: skip the butterflies (memory-pipeline ceiling measurement, results are garbage)
                          // L2 eviction hints on the TMA copies -- bit 1: input loads evict-first, bit 2: ring loads evict-first,
                          // bit 3: ring stores evict-last, bit 4: output stores evict-first
    };
};

// pipeline trace (tools/fused_trace.py): FUSED_TRACE_CTAS CTAs x 4 roles (producer, storer, consumer group 0 / 1) x
// FUSED_TRACE_WORDS stamps, each (globaltimer << 8) | event tag; the last word of a role's region = number of stamps
static constexpr uint32_t FUSED_TRACE_CTAS = 16, FUSED_TRACE_WORDS = 4096;
inline uint64_t fused_trace_bytes() { return (uint64_t)FUSED_TRACE_CTAS * 4 * FUSED_TRACE_WORDS * 8; }

#if defined(__CUDACC__)
struct FusedTrace {
    unsigned long long* base;  // null: off
    uint32_t n;
    B2_D void init(unsigned long long* trace, int role) {
        base = (trace != nullptr && blockIdx.x < FUSED_TRACE_CTAS) ? trace + ((size_t)blockIdx.x * 4 + role) * FUSED_TRACE_WORDS : nullptr;
        n = 0;
    }
    B2_D void stamp(uint32_t tag) {
        if (base != nullptr && n + 1 < FUSED_TRACE_WORDS) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            base[n++] = (t << 8) | tag;
        }
    }
    B2_D void finish() {
        if (base != nullptr) base[FUSED_TRACE_WORDS - 1] = n;
    }
};
// counter += 1 with release semantics at device scope: everything this thread did (or observed through a barrier) before
// is visible to whoever acquires the new value
B2_D void red_release_add1(uint32_t* p) { asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory"); }
B2_D uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// spin until *ctr >= target (bounded: a scheduling bug raises the error flag instead of hanging the GPU)
B2_D void fused_spin(uint32_t* ctl, const uint32_t* ctr, uint32_t target) {
    uint32_t spins = 0;
    while (ld_acquire_u32(ctr) < target) {
        __nanosleep(spins < 64 ? 20 : 200);
        if (++spins > (1u << 22) || (spins > 4096 && ld_relaxed_u32(ctl + 1) != 0)) {
            atomicExch(ctl + 1, 1u);
            break;
        }
    }
}

// the phases of one tile inside a consumer group (named barrier `bar_id` among KT::NT threads); the last phase of
// TmaTileKernel (the store) belongs to the storer thread.
// `release`: direct-output tiles (Params::direct) hand their stage back to the producer as soon as the last exchange has
// been read -- the barrier that follows phase NPHASE - 3 -- i.e. before the last butterflies and the global stores.
template <class KT, int P>
struct GroupPhases {
    static B2_D void run(const typename KT::Params& p, uint32_t bid, int ltid, typename KT::Regs& r, cx<typename KT::T>* buf, int bar_id,
                         uint64_t* release) {
        KT::template phase<P>(p, bid, ltid, r, buf);
        if constexpr (P + 2 < KT::NPHASE) {
            tma::named_bar_sync(bar_id, KT::NT);
            if constexpr (P + 3 == KT::NPHASE) {
                if (release != nullptr && ltid == 0) tma::mbar_arrive(release);
            }
            GroupPhases<KT, P + 1>::run(p, bid, ltid, r, buf, bar_id, release);
        }
    }
};

template <class KA, class KB, int NG, int NS>
__global__ void __launch_bounds__(FusedKernel<KA, KB, NG, NS>::NT, 1)
run_fused(const __grid_constant__ typename FusedKernel<KA, KB, NG, NS>::Params p) {
    using FK = FusedKernel<KA, KB, NG, NS>;
    using C = cx<typename FK::T>;
    constexpr int NTG = FK::NTG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned char* base = smem_raw + ((128u - (tma::smem_u32(smem_raw) & 127u)) & 127u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + (size_t)NS * FK::STAGE_BYTES);
    uint64_t* full = bars;            // tile landed (producer arrival + TMA bytes)
    uint64_t* meta = bars + NS;       // tile description written (consumers may prefetch their tables)
    uint64_t* outf = bars + 2 * NS;   // finished tile in the buffer (one arrival per consumer warp)
    uint64_t* empty = bars + 3 * NS;  // the store has read the buffer (storer)
    uint64_t* q_full = bars + 4 * NS;             // scheduler -> producer queue
    uint64_t* q_empty = bars + 4 * NS + FK::NQ;
    volatile uint32_t* info = reinterpret_cast<volatile uint32_t*>(bars + 4 * NS + 2 * FK::NQ);  // [stage][4]: kind (0 A, 1 B, 2 end), tile, slot
    volatile uint32_t* qent = info + 4 * NS;      // [queue slot][4]: the same triple
    const int tid = (int)threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const FlowSched& sc = p.sched;
    uint32_t* ready = p.ctl + FLOW_CTL_HEAD;
    uint32_t* freed = ready + sc.ring_w;
    if (tid == 0) {
        for (int s = 0; s < NS; ++s) {
            tma::mbar_init(&full[s], 1);
            tma::mbar_init(&meta[s], 1);
            tma::mbar_init(&outf[s], NTG / 32);
            tma::mbar_init(&empty[s], 1);
        }
        for (int q = 0; q < FK::NQ; ++q) {
            tma::mbar_init(&q_full[q], 1);
            tma::mbar_init(&q_empty[q], 1);
        }
        tma::fence_mbar_init();
    }
    __syncthreads();
    auto stage_buf = [&](uint32_t s) { return reinterpret_cast<C*>(base + (size_t)s * FK::STAGE_BYTES); };
    // tiles the scheduler may run ahead of the producer: 1 (measured best: a ticket claimed early is a tile others may wait for)
    const uint32_t nq = (p.flags & 64u) ? (uint32_t)FK::NQ : 1u;

    if (warp >= FK::SVC_WARP) {
        // each budget change sits inside its branch, so that ptxas allocates every role's code under that role's budget
        tma::setmaxnreg_dec<FK::SVC_REGS>();
        if (warp == FK::SVC_WARP + 2) {
            // ---------------- scheduler ----------------
            // Draws tickets, resolves their dependencies and hands ready-to-load tiles to the producer through a small queue.
            // Everything with a round trip to L2 in it (ticket counter, dependency counters) lives in THIS thread: measured with
            // the pipeline trace (tools/fused_trace.py), the same work inside the producer thread kept a freed stage empty for 1.4 us.
            if (lane == 0) {
                uint32_t k = 0;
                uint32_t ticket = atomicAdd(p.ctl, 1u);
                while (ticket < sc.total) {
                    int kind;
                    uint32_t t, tile;
                    bool valid;
                    sc.decode(ticket, kind, t, tile, valid);
                    const uint32_t next = atomicAdd(p.ctl, 1u);  // in flight while this ticket's dependency is resolved
                    if (valid) {
                        const FlowDep d = flow_dep(sc, p.ctl, ticket);
                        if (d.ptr != nullptr && ld_acquire_u32(d.ptr) < d.target) fused_spin(p.ctl, d.ptr, d.target);
                        // the acquire above (generic proxy) -> the TMA accesses of the slot (async proxy), issued by the producer and the
                        // storer after they have synchronised with this thread through the queue.  The fence sits HERE because in the
                        // producer it also waited for that thread's outstanding tile loads (measured: +0.7..1.1 us per tile).
                        if (d.ptr != nullptr) tma::fence_proxy_async_all();
                        const uint32_t q = k % nq, qph = (k / nq) & 1u;
                        tma::mbar_wait(&q_empty[q], qph ^ 1u);
                        qent[4 * q + 0] = (uint32_t)kind;
                        qent[4 * q + 1] = kind == 0 ? t * sc.TA + tile : t * sc.TB + tile;
                        qent[4 * q + 2] = t % sc.ring_w;
                        tma::mbar_arrive(&q_full[q]);
                        ++k;
                    }
                    ticket = next;
                }
                const uint32_t q = k % nq, qph = (k / nq) & 1u;
                tma::mbar_wait(&q_empty[q], qph ^ 1u);
                qent[4 * q + 0] = 2u;  // end of work
                tma::mbar_arrive(&q_full[q]);
            }
        } else if (warp == FK::SVC_WARP) {
            // ---------------- producer ----------------
            if (lane == 0) {
                uint32_t i = 0;
                FusedTrace tr;
                tr.init(p.trace, 0);
                const unsigned long long pol_a = (p.flags & 2u) ? l2_evict_first() : 0ull, pol_b = (p.flags & 4u) ? l2_evict_first() : 0ull;
                for (uint32_t k = 0;; ++k) {
                    const uint32_t q = k % nq, qph = (k / nq) & 1u;
                    tma::mbar_wait(&q_full[q], qph);
                    const uint32_t kind = qent[4 * q + 0], bid = qent[4 * q + 1], slot = qent[4 * q + 2];
                    tma::mbar_arrive(&q_empty[q]);
                    if (kind == 2u) break;
                    const uint32_t s = i % NS, ph = (i / NS) & 1u;
                    tr.stamp(0x10u | kind);              // a resolved ticket in hand
                    tma::mbar_wait(&empty[s], ph ^ 1u);  // (passes at once for the first NS tiles)
                    tr.stamp(0x20u | s);                 // stage free
                    info[4 * s + 0] = kind;
                    info[4 * s + 1] = bid;
                    info[4 * s + 2] = slot;
                    tma::mbar_arrive(&meta[s]);
                    if (kind == 0u)
                        KA::issue_load(p.a, bid, stage_buf(s), &full[s], pol_a);
                    else
                        KB::issue_load(p.b, bid, stage_buf(s), &full[s], pol_b);
                    tr.stamp(0x30u | s);  // load queued
                    ++i;
                }
                for (int g = 0; g < NG; ++g, ++i) {  // one end marker per consumer group
                    const uint32_t s = i % NS, ph = (i / NS) & 1u;
                    tma::mbar_wait(&empty[s], ph ^ 1u);
                    info[4 * s + 0] = 2u;
                    tma::mbar_arrive(&meta[s]);
                }
                tr.finish();
            }
        } else if (warp == FK::SVC_WARP + 1) {
            // ---------------- storer ----------------
            // Finished tiles that leave through shared memory (all pass-B tiles; pass-A tiles too when the ring is not tile-major)
            // complete their stage's `outf` barrier in no particular order: poll the stages.
            if (lane == 0) {
                uint32_t* pending = nullptr;  // ready counter of the last pass-A tile stored, not yet published
                const unsigned long long pol_a = (p.flags & 8u) ? l2_evict_last() : 0ull, pol_b = (p.flags & 16u) ? l2_evict_first() : 0ull;
                FusedTrace tr;
                tr.init(p.trace, 1);
                uint32_t sph = 0;  // bit s: parity of the next completion of outf[s]
                uint32_t held = 0xffffffffu;  // stage whose store is queued but not yet known to have been read (two-in-flight mode)
                int ends = 0;
                uint32_t idle = 0;
                while (ends < NG) {
                    bool any = false;
                    for (uint32_t s = 0; s < (uint32_t)NS; ++s) {
                        if (!tma::mbar_test(&outf[s], (sph >> s) & 1u)) continue;
                        sph ^= 1u << s;
                        any = true;
                        const uint32_t kind = info[4 * s + 0], bid = info[4 * s + 1], slot = info[4 * s + 2];
                        if (kind == 2u) {
                            ++ends;
                            continue;
                        }
                        tr.stamp(0x40u | s);  // finished tile seen
                        if (kind == 0u)
                            KA::issue_store(p.a, bid, stage_buf(s), pol_a);
                        else
                            KB::issue_store(p.b, bid, stage_buf(s), pol_b);
                        tma::bulk_commit();
                        if (pending != nullptr) {  // every group but the one just committed has completed
                            tma::bulk_wait<1>();
                            tma::fence_proxy_async_all();
                            red_release_add1(pending);
                            pending = nullptr;
                        }
                        tr.stamp(0x50u | s);       // store queued (+ previous pass-A tile published)
                        if (p.flags & 128u) {
                            // keep the store engine fed: the previous store's stage is released once this one is queued behind it
                            if (held != 0xffffffffu) {
                                tma::bulk_wait_read<1>();
                                tma::mbar_arrive(&empty[held]);
                                tr.stamp(0x60u | held);
                            }
                            held = s;
                        } else {
                            tma::bulk_wait_read<0>();  // the buffer may be refilled
                            tma::mbar_arrive(&empty[s]);
                            tr.stamp(0x60u | s);  // stage released
                        }
                        if (kind == 0u) pending = ready + slot;
                    }
                    if (!any) {
                        if (held != 0xffffffffu) {
                            tma::bulk_wait_read<0>();
                            tma::mbar_arrive(&empty[held]);
                            tr.stamp(0x60u | held);
                            held = 0xffffffffu;
                        }
                        if (pending != nullptr) {  // idle: other CTAs (or this CTA's own scheduler) may be waiting for that tile
                            tma::bulk_wait<0>();
                            tma::fence_proxy_async_all();
                            red_release_add1(pending);
                            pending = nullptr;
                        }
                        __nanosleep(idle < 8 ? 32 : 128);
                        ++idle;
                    } else {
                        idle = 0;
                    }
                }
                tma::bulk_wait<0>();
                if (pending != nullptr) {
                    tma::fence_proxy_async_all();
                    red_release_add1(pending);
                }
                tr.finish();
            }
        }  // warp SVC_WARP + 3 only completes the warpgroup
    } else {
        tma::setmaxnreg_inc<FK::CONS_REGS>();
        // ---------------- consumers ----------------
        const int g = warp / (NTG / 32);
        const int ltid = tid - g * NTG;
        const int bar_id = 1 + g;
        constexpr bool DA = KA::DIRECT_OUT;  // pass-A results go from the registers to the tile-major ring
        constexpr bool DB = KB::DIRECT_OUT;  // pass-B results go from the registers to the caller's output
        FusedTrace tr;
        tr.init(ltid == 0 ? p.trace : nullptr, 2 + (g & 1));
        for (uint32_t i = (uint32_t)g;; i += NG) {
            const uint32_t s = i % NS, ph = (i / NS) & 1u;
            tma::mbar_wait(&meta[s], ph);
            tr.stamp(0x70u | s);  // tile description seen
            const uint32_t kind = info[4 * s + 0], bid = info[4 * s + 1], slot = info[4 * s + 2];
            C* buf = stage_buf(s);
            bool via_smem = true;  // the finished tile sits in the stage buffer and leaves through the storer
            if (kind == 0u) {
                typename KA::Regs r;
                KA::prefetch(p.a, bid, ltid, r);  // table loads overlap the tile's flight
                tma::mbar_wait(&full[s], ph);
                tr.stamp(0x80u | s);  // tile landed
                if (!(p.flags & 1u)) {
                    GroupPhases<KA, 0>::run(p.a, bid, ltid, r, buf, bar_id, DA ? &empty[s] : nullptr);
                    if constexpr (DA) {
                        // count the tile as landed once every thread of the group has issued its stores, with a release that
                        // covers them (barrier + release by one thread: the pattern of a split-K semaphore)
                        tma::named_bar_sync(bar_id, NTG);
                        if (ltid == 0) red_release_add1(ready + slot);
                        via_smem = false;
                    }
                } else if (DA) {
                    if (ltid == 0) {
                        tma::mbar_arrive(&empty[s]);
                        red_release_add1(ready + slot);
                    }
                    via_smem = false;
                } else {
                    tma::fence_proxy_async();
                }
            } else if (kind == 1u) {
                typename KB::Regs r;
                KB::prefetch(p.b, bid, ltid, r);
                tma::mbar_wait(&full[s], ph);
                tr.stamp(0x80u | s);
                if (!(p.flags & 1u)) {
                    GroupPhases<KB, 0>::run(p.b, bid, ltid, r, buf, bar_id, DB ? &empty[s] : nullptr);
                    if constexpr (DB) via_smem = false;  // the stage was handed back after the last exchange read
                } else if (DB) {
                    if (ltid == 0) tma::mbar_arrive(&empty[s]);
                    via_smem = false;
                } else {
                    tma::fence_proxy_async();
                }
            }
            if (via_smem) {
                // every thread has written its share of the dense output tile and fenced it towards the async proxy
                __syncwarp();
                if (lane == 0) tma::mbar_arrive(&outf[s]);
            }
            tr.stamp(0x90u | s);  // tile done (this thread)
            // pass-B tile: its ring-slot rows are consumed (every thread loaded its inputs and issued its discards at least two
            // group barriers ago).  Published here, at the end of the tile, so the release never sits between two barriers.
            if (kind == 1u && ltid == 0) red_release_add1(freed + slot);
            if (kind == 2u) break;
        }
        tr.finish();
    }
}
#endif

}  // namespace b2
