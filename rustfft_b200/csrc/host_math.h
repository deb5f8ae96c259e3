// Host-side mathematics of the planner: exact-ish twiddles, integer helpers, and a long-double
// reference FFT used ONLY at plan time to precompute the frequency-domain multipliers of
// Bluestein's and Rader's algorithms (the reference runs its own inner FFT for that,
// src/algorithm/bluesteins_algorithm.rs:62-83, src/algorithm/raders_algorithm.rs:86-109).
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

#include "common.h"

namespace b2 {
namespace hm {

typedef long double ld;
struct cld { ld x, y; };

// cos / sin of the angle o pi/4 + (flip ? pi/4 - t : t), 0 <= t <= pi/4, from cosl / sinl of t
inline void octant_sincos(unsigned o, bool flip, ld t, ld& c, ld& s) {
    const ld ct = cosl(t), st = sinl(t);
    const ld cphi = flip ? st : ct, sphi = flip ? ct : st;
    switch (o >> 1) {
        case 0: c = cphi; s = sphi; break;
        case 1: c = -sphi; s = cphi; break;
        case 2: c = -cphi; s = -sphi; break;
        default: c = sphi; s = -cphi; break;
    }
}

// cos(2*pi*k/n), sin(2*pi*k/n): integer octant reduction, then cosl/sinl on [0, pi/4].
// Contract of src/twiddles.rs:6-23 (evaluate in higher precision, round once to T) -- here the
// evaluation is 64-bit-mantissa long double with an exactly reduced argument.
inline void sincos_2pi(uint64_t k, uint64_t n, ld& c, ld& s) {
    k %= n;
    const unsigned __int128 k8 = (unsigned __int128)k * 8u;
    const unsigned o = (unsigned)(k8 / n);
    const uint64_t r = (uint64_t)(k8 % n);
    const bool flip = (o & 1u) != 0;
    const ld quarter_pi = 0.785398163397448309615660845819875721L;
    const ld t = (flip ? (ld)(n - r) : (ld)r) / (ld)n * quarter_pi;
    octant_sincos(o, flip, t, c, s);
}

// forward twiddle exp(-2*pi*i*k/n)
inline cld twiddle_ld(uint64_t k, uint64_t n) {
    ld c, s;
    sincos_2pi(k, n, c, s);
    return cld{c, -s};
}
template <typename T> inline cx<T> twiddle(uint64_t k, uint64_t n) {
    cld w = twiddle_ld(k, n);
    return mk<T>((T)w.x, (T)w.y);
}

// Phases of the chirp-z tables (impl.inl, czt_tables), in turns, reduced mod 1 exactly and kept as fixed-point fractions of
// PHASE_BITS bits.  A finite double is m 2^e with |m| < 2^53, so v k for k < 2^62 (t^2 with t < 2^31) is the 115-bit integer m k
// times a power of two: the integer turns drop out exactly, and only bits below 2^-124 turns are cut.  Evaluating the phase in
// double instead would lose |v k| ulps of a turn, which grows with k^2 along a chirp.
static constexpr int PHASE_BITS = 124;
typedef unsigned __int128 u128;
static constexpr u128 PHASE_ONE = (u128)1 << PHASE_BITS;
// frac(v k 2^sh) in units of 2^-PHASE_BITS turns (v finite, k < 2^62, sh small)
inline u128 frac_turns(double v, uint64_t k, int sh) {
    if (v == 0 || k == 0) return 0;
    int e;
    const double fr = std::frexp(v, &e);
    const int64_t m = (int64_t)std::ldexp(fr, 53);  // v = m 2^(e - 53), exactly
    const int s = e - 53 + sh + PHASE_BITS;          // v k = (|m| k) 2^s units
    const u128 a = (u128)(m < 0 ? -m : m) * k;
    u128 r = 0;
    if (s >= PHASE_BITS) r = 0;                       // whole turns
    else if (s >= 0) r = (a << s) & (PHASE_ONE - 1);  // (mod 2^128, then mod 2^124: exact)
    else if (s > -128) r = a >> -s;                   // below 2^-124 turns: cut
    return m < 0 ? (PHASE_ONE - r) & (PHASE_ONE - 1) : r;
}
// exp(-2 pi i phase) for a phase of `num` units of 2^-PHASE_BITS turns: octant reduction on the integer, cosl / sinl on
// [0, pi/4], one rounding to long double (the contract of sincos_2pi)
inline cld turns_twiddle_ld(u128 num) {
    num &= PHASE_ONE - 1;
    const u128 eighth = PHASE_ONE >> 3;
    const unsigned o = (unsigned)(num >> (PHASE_BITS - 3));
    const u128 r = num & (eighth - 1);
    const bool flip = (o & 1u) != 0;
    const ld quarter_pi = 0.785398163397448309615660845819875721L;
    const ld t = ldexpl((ld)(flip ? eighth - r : r), -(PHASE_BITS - 3)) * quarter_pi;
    ld c, s;
    octant_sincos(o, flip, t, c, s);
    return cld{c, -s};
}

inline cld mul(cld a, cld b) { return cld{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }

// in-place forward FFT, power-of-two length, long double
inline void fft_pow2_ld(std::vector<cld>& a) {
    const size_t n = a.size();
    if (n < 2) return;
    for (size_t i = 1, j = 0; i < n; ++i) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) { cld t = a[i]; a[i] = a[j]; a[j] = t; }
    }
    for (size_t len = 2; len <= n; len <<= 1) {
        std::vector<cld> w(len / 2);
        for (size_t k = 0; k < len / 2; ++k) w[k] = twiddle_ld(k, len);
        for (size_t i = 0; i < n; i += len)
            for (size_t k = 0; k < len / 2; ++k) {
                cld u = a[i + k], v = mul(a[i + k + len / 2], w[k]);
                a[i + k] = cld{u.x + v.x, u.y + v.y};
                a[i + k + len / 2] = cld{u.x - v.x, u.y - v.y};
            }
    }
}

// forward FFT of any length whose prime factors are small, long double: recursive decimation in time by the smallest
// prime factor r of the length (r interleaved sub-transforms, then r-point DFTs across them).  Plan-time only: the
// multipliers of Rader / Bluestein plans over smooth inner lengths.
inline void fft_any_ld_rec(const cld* in, size_t stride, cld* out, size_t n, const std::vector<cld>& wn, size_t wstep) {
    if (n == 1) {
        out[0] = in[0];
        return;
    }
    size_t r = 2;
    while (n % r) ++r;
    const size_t m = n / r;
    for (size_t j = 0; j < r; ++j) fft_any_ld_rec(in + j * stride, stride * r, out + j * m, m, wn, wstep * r);
    std::vector<cld> t(r);
    for (size_t k = 0; k < m; ++k) {
        for (size_t j = 0; j < r; ++j) t[j] = mul(out[j * m + k], wn[(j * k * wstep) % wn.size()]);
        for (size_t q = 0; q < r; ++q) {
            cld acc{0, 0};
            for (size_t j = 0; j < r; ++j) {
                const cld v = mul(t[j], wn[(j * q * m * wstep) % wn.size()]);
                acc.x += v.x;
                acc.y += v.y;
            }
            // (out[q m + k] for all q are read above before any is written: t[] holds them)
            out[q * m + k] = acc;
        }
    }
}
inline void fft_any_ld(std::vector<cld>& a) {
    const size_t n = a.size();
    if (n < 2) return;
    std::vector<cld> wn(n), out(n);
    for (size_t k = 0; k < n; ++k) wn[k] = twiddle_ld(k, n);
    fft_any_ld_rec(a.data(), 1, out.data(), n, wn, 1);
    a.swap(out);
}

inline bool is_pow2(uint64_t n) { return n && !(n & (n - 1)); }
inline uint32_t ilog2(uint64_t n) {
    uint32_t l = 0;
    while ((1ull << (l + 1)) <= n) ++l;
    return l;
}
inline uint64_t next_pow2(uint64_t n) {
    uint64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}
inline bool is_prime(uint64_t n) {
    if (n < 2) return false;
    for (uint64_t d = 2; d * d <= n; ++d)
        if (n % d == 0) return false;
    return true;
}
inline uint64_t mulmod(uint64_t a, uint64_t b, uint64_t m) { return (uint64_t)((unsigned __int128)a * b % m); }
inline uint64_t powmod(uint64_t b, uint64_t e, uint64_t m) {
    uint64_t r = 1 % m;
    b %= m;
    while (e) {
        if (e & 1) r = mulmod(r, b, m);
        b = mulmod(b, b, m);
        e >>= 1;
    }
    return r;
}
inline uint64_t gcd(uint64_t a, uint64_t b) {
    while (b) {
        const uint64_t t = a % b;
        a = b;
        b = t;
    }
    return a;
}
// a^-1 mod m (gcd(a, m) = 1, m > 1), extended Euclid
inline uint64_t invmod(uint64_t a, uint64_t m) {
    __int128 t = 0, nt = 1, r = (__int128)m, nr = (__int128)(a % m);
    while (nr != 0) {
        const __int128 q = r / nr;
        __int128 x = t - q * nt;
        t = nt;
        nt = x;
        x = r - q * nr;
        r = nr;
        nr = x;
    }
    if (t < 0) t += (__int128)m;
    return (uint64_t)t;
}
inline uint64_t largest_prime_factor(uint64_t n) {
    uint64_t best = 1;
    for (uint64_t d = 2; d * d <= n; ++d)
        while (n % d == 0) {
            best = d;
            n /= d;
        }
    return n > 1 ? n : best;
}
// smallest primitive root of prime p (same choice as src/math_utils.rs:3-20)
inline uint64_t primitive_root(uint64_t p) {
    std::vector<uint64_t> fac;
    uint64_t m = p - 1;
    for (uint64_t d = 2; d * d <= m; ++d)
        if (m % d == 0) {
            fac.push_back(d);
            while (m % d == 0) m /= d;
        }
    if (m > 1) fac.push_back(m);
    for (uint64_t g = 2; g < p; ++g) {
        bool ok = true;
        for (uint64_t f : fac)
            if (powmod(g, (p - 1) / f, p) == 1) { ok = false; break; }
        if (ok) return g;
    }
    return 0;
}

}  // namespace hm
}  // namespace b2
