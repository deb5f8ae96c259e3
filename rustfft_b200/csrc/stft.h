// Short-time Fourier transforms of real rows (b200fft_stft_*).  A plan fixes a real window w of N = n_fft taps (N even), the hop,
// the signal length n and `center`; frame f of a row x starts at padded sample f hop:
//     xp = center ? reflect-pad(x, N/2 on each side) : x         (torch's pad_mode="reflect": xp[-i] = x[i], xp[n-1+i] = x[n-1-i])
//     S[f][k] = sum_u w[u] xp[f hop + u] W_N^(k u),   k = 0 .. N/2                       (unnormalised; frame-major output)
//     y[t] = sum_f w[u] irfft(S[f])[u] / env[t + s],   u = t + s - f hop,   env[p] = sum_f w[p - f hop]^2,   s = center ? N/2 : 0
// The inverse is the least-squares inverse (torch.istft with length = n): the division by the window envelope is part of it, and the
// 1/N of the inverse FFT folds into the same table entry 1/(N env), evaluated on the host in long double and rounded once.
//
// StftKernel<G>: the whole forward of N = 2M points (M = G::L, a power of two) in one CTA pass; the G::F engine slots of a CTA hold F
// consecutive frames of one row (a CTA never straddles two rows: a row whose frame count is not a multiple of F leaves idle slots in its
// last CTA, whose results are not stored).
//   load:     the span of the CTA's frames, (F' - 1) hop + N reals (F' <= F frames), coalesced into shared memory once; the reflect
//             map is applied per element, and only in CTAs whose span leaves [0, n)
//   build:    z[m] = w[2m] s[f hop + 2m] + i w[2m+1] s[f hop + 2m + 1]       (the window through ldg, as M complex pairs)
//   engine:   the M-point FFT
//   combine:  Z to shared memory; the pair (k, M-k) gives X[k] = E[k] + W_N^k O[k] (real.h's unpack), folded into two table entries
//             per k: X[k] = A_k Z[k] + B_k conj Z[M-k], A_k = (1 - i W_N^k) / 2, B_k = (1 + i W_N^k) / 2; X[0] and X[M] are
//             Re Z[0] + Im Z[0] and Re Z[0] - Im Z[0]
//   store:    X into shared memory at f (M + 1) + k, then one contiguous run of F' (M + 1) complex values
// One read of the signal (plus the halo between neighbouring CTAs) and one write of the spectrum; no workspace.
//
// StftFrameKernel<T>: the general forward's framing: the reflect pad, the framing and the window into a workspace of [frames][N] reals,
// one thread per workspace element; the real plan of N points then runs over the frames straight into the output.
// IstftOlaKernel<T>: the inverse's overlap-add after the real plan's inverse over every frame (frames [frames][N], unnormalised: N
// times irfft): one thread per output sample t, which sums w[u] frame_f[u] over the frames f covering t + s in increasing f (a fixed
// order: repeats are bit-identical, no atomics) and multiplies by the table entry 1/(N env[t + s]) (zero past the covered span).
#pragma once
#include "kernels.h"
#include "conv.h"

namespace b2 {

// sample idx of a row of n samples, reflected at both ends (|idx| < n - 1 past an end: one fold)
B2_HD int32_t stft_reflect(int32_t i, int32_t n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

template <class G>
struct StftKernel {
    using T = typename G::T;
    using Eng = Engine<G, JF, JF>;
    static constexpr int M = G::L, N = 2 * G::L, F = G::F, NT = G::NT;
    static constexpr int MIN_BLOCKS = default_min_blocks(G::NT, 32);
    static constexpr int P_ENG = 2;                         // phase 0: load, 1: build, then the engine
    static constexpr int P_LAST = P_ENG + Eng::NPHASE - 1;  // last engine phase
    static constexpr int NPHASE = P_LAST + 4;               // combine: Z to shared memory, X in registers, X to shared memory, store
    static constexpr size_t SMEM_BYTES = sizeof(cx<T>) * (size_t)G::F * G::LP;
    static_assert((M & (M - 1)) == 0 && M >= 2, "M must be a power of two");
    static_assert(G::LP >= M + 1, "a frame's M + 1 bins must fit its slot of the engine's buffer");
    struct Params {
        const T* in;      // rows of n samples
        cx<T>* out;       // rows of frames * (M + 1) bins
        const cx<T>* win; // the window as M pairs (w[2m], w[2m+1])
        const cx<T>* ta;  // A_k, k < M
        const cx<T>* tb;  // B_k, k < M
        const cx<T>* tw;  // stage twiddles of the M-point FFT
        uint32_t n, frames, hop, pad;  // signal length, frames per row, hop, left padding (center: N/2, else 0)
        FastDiv div_cpr;  // by CTAs per row
        uint32_t rows;    // rows in this launch
    };
    struct Regs { cx<T> v[G::E]; };

    // row, first frame and frames of this CTA
    static B2_HD void locate(const Params& p, uint32_t bid, uint32_t& row, uint32_t& f0, uint32_t& nf) {
        row = p.div_cpr.div(bid);
        f0 = (bid - row * p.div_cpr.d) * F;
        nf = p.frames - f0 < (uint32_t)F ? p.frames - f0 : (uint32_t)F;
    }

    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs& r, cx<T>* smem) {
        int f, j;
        tid_to_fj<G, JF>(tid, f, j);
        T* s = reinterpret_cast<T*>(smem);
        if constexpr (P == 0) {
            uint32_t row, f0, nf;
            locate(p, bid, row, f0, nf);
            const int32_t span = (int32_t)((nf - 1) * p.hop) + N, base = (int32_t)(f0 * p.hop) - (int32_t)p.pad, n = (int32_t)p.n;
            const T* x = p.in + (size_t)row * p.n;
            // (loops with a run-time bound: fully unrolled, the f32 M = 16384 kernel spilled)
            if (base >= 0 && base + span <= n) {
                for (int32_t e = tid; e < span; e += NT) s[e] = ld_stream_r(x + base + e);
            } else {  // the first or last CTA of a centred row: reflect per element
                for (int32_t e = tid; e < span; e += NT) s[e] = ld_stream_r(x + stft_reflect(base + e, n));
            }
        }
        if constexpr (P == 1) {
            const T* fr = s + f * p.hop;
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int m = j + G::TP * q;
                const cx<T> w = ldg(p.win + m);
                r.v[q] = mk<T>(w.x * fr[2 * m], w.y * fr[2 * m + 1]);
            }
        }
        if constexpr (P >= P_ENG && P <= P_LAST) Eng::template phase<P - P_ENG>(tid, r.v, smem, p.tw);
        if constexpr (P == P_LAST) {
            // the engine's last phase reads no shared memory: the frames can be overwritten now
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) smem[f * M + j + G::TP * q] = r.v[q];
        }
        if constexpr (P == P_LAST + 1) {
            // (Z[k] read back from shared memory, not kept in registers: holding it next to the table loads made f32 M = 16384 spill)
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                const cx<T> zk = smem[f * M + k];
                if (q == 0 && j == 0) {
                    r.v[q] = mk<T>(zk.x + zk.y, zk.x - zk.y);  // X[0], X[M]
                } else {
                    const cx<T> zm = conj(smem[f * M + M - k]);
                    r.v[q] = cmul(zk, ldg(p.ta + k)) + cmul(zm, ldg(p.tb + k));
                }
            }
        }
        if constexpr (P == P_LAST + 2) {
            B2_UNROLL
            for (int q = 0; q < G::E; ++q) {
                const int k = j + G::TP * q;
                if (q == 0 && j == 0) {
                    smem[f * (M + 1)] = mk<T>(r.v[q].x, (T)0);
                    smem[f * (M + 1) + M] = mk<T>(r.v[q].y, (T)0);
                } else {
                    smem[f * (M + 1) + k] = r.v[q];
                }
            }
        }
        if constexpr (P == NPHASE - 1) {
            uint32_t row, f0, nf;
            locate(p, bid, row, f0, nf);
            cx<T>* dst = p.out + (size_t)(row * p.frames + f0) * (M + 1);
            const uint32_t cnt = nf * (M + 1);
            for (uint32_t i = tid; i < cnt; i += NT) st_stream(dst + i, smem[i]);
        }
    }
};

// general forward: workspace element i = g N + u (g < frames of this launch) is w[u] xp[(fr0 + g) hop + u] of its row
template <typename TT>
struct StftFrameKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const T* in;       // the launch's first row
        T* out;            // [cnt][N]
        const T* win;      // N taps
        uint64_t n_elem;   // cnt * N
        uint32_t n, hop, pad, fr0;  // signal length, hop, left padding, frame (in its row) of the launch's first frame
        FastDiv div_n;      // by N
        FastDiv div_frames; // by frames per row
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t g = p.div_n.div((uint32_t)i), u = (uint32_t)i - g * p.div_n.d;
        const uint32_t t = p.fr0 + g, row = p.div_frames.div(t), f = t - row * p.div_frames.d;
        const int32_t idx = stft_reflect((int32_t)(f * p.hop + u) - (int32_t)p.pad, (int32_t)p.n);
        p.out[i] = p.win[u] * p.in[(size_t)row * p.n + idx];
    }
};

// inverse overlap-add: output sample t of row `row` of the launch, from the N-point frames of the launch's rows ([rows][frames][N])
template <typename TT>
struct IstftOlaKernel {
    using T = TT;
    static constexpr int NT = 256;
    static constexpr int MIN_BLOCKS = 4;
    static constexpr int NPHASE = 1;
    static constexpr size_t SMEM_BYTES = 0;
    struct Params {
        const T* in;       // frames of the launch's rows
        T* out;            // rows of n samples
        const T* win;      // N taps
        const T* inv;      // n entries: 1 / (N env[t + s]), 0 past the covered span
        uint64_t n_elem;   // rows * n
        uint32_t frames, N, s;
        FastDiv div_n;     // by the signal length n
        FastDiv div_hop;   // by the hop
    };
    struct Regs {};
    template <int P>
    static B2_HD void phase(const Params& p, uint32_t bid, int tid, Regs&, cx<T>*) {
        const uint64_t i = (uint64_t)bid * NT + tid;
        if (i >= p.n_elem) return;
        const uint32_t row = p.div_n.div((uint32_t)i), t = (uint32_t)i - row * p.div_n.d, pos = t + p.s, hop = p.div_hop.d;
        const uint32_t last = p.div_hop.div(pos), f_hi = last < p.frames - 1 ? last : p.frames - 1;
        const uint32_t f_lo = pos >= p.N ? p.div_hop.div(pos - p.N) + 1 : 0;
        const T* fr = p.in + (size_t)row * p.frames * p.N;
        T sum = (T)0;
        for (uint32_t f = f_lo; f <= f_hi; ++f) {
            const uint32_t u = pos - f * hop;
            sum += p.win[u] * fr[(size_t)f * p.N + u];
        }
        p.out[i] = sum * p.inv[t];
    }
};

}  // namespace b2
