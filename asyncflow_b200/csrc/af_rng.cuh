// AF-RNG, device side: Philox4x32-10 counter-based variates for the replica engine.
//
// Replaces numpy.random.Generator on the hot path: rng.uniform() / general_sampler
// at reference runtime/actors/edge.py:78,90, rng.integers at
// runtime/actors/server.py:101, rng.poisson / rng.normal / rng.random in
// samplers/{poisson_poisson,gaussian_poisson}.py via samplers/common_helpers.py.
// The normative statement of the number streams is oracle/afrng.py; this header
// is an independent restatement and is checked against it bit for bit
// (tests/test_gpu_rng.py on the device, tests/test_host_twin.py on the host).
//
// Bit-exactness contract: only IEEE double + - * / sqrt in a fixed order, no
// FMA contraction -- compile with nvcc -fmad=false (and gcc -ffp-contract=off
// for the host twin).
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>
#include "../../include/asyncflow_b200.h"

#if defined(__CUDACC__)
#define AF_HD __host__ __device__ __forceinline__
#define AF_HD_NOINLINE __host__ __device__ __noinline__
#else
#define AF_HD inline
#define AF_HD_NOINLINE inline
#endif

namespace afr {

constexpr uint32_t P_GEN = 0u, P_EDGE = 1u, P_SERVER = 2u;

struct U4 { uint32_t x, y, z, w; };

AF_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// (one shared body: Philox and log are used from four places; see the code-size rule in af_core.cuh)
AF_HD_NOINLINE U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = mulhi32(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        uint32_t hi1 = mulhi32(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        U4 n;
        n.x = hi1 ^ c.y ^ k0;
        n.y = lo1;
        n.z = hi0 ^ c.w ^ k1;
        n.w = lo0;
        c = n;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

AF_HD double u53(uint32_t hi, uint32_t lo) {
    return (double)(((uint64_t)(hi >> 5) << 26) + (uint64_t)(lo >> 6)) * (1.0 / 9007199254740992.0);
}
AF_HD double s32(uint32_t w) { return ((double)w + 0.5) * (1.0 / 2147483648.0) - 1.0; }

AF_HD uint64_t d2u(double x) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t b; memcpy(&b, &x, 8); return b;
#endif
}
AF_HD double u2d(uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)b);
#else
    double x; memcpy(&x, &b, 8); return x;
#endif
}
AF_HD double af_sqrt(double x) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(x);
#else
    return sqrt(x);
#endif
}
AF_HD double af_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// The latency histogram's bin of `lat` (AF_HIST_BINS log-linear bins, clamped at both ends): the per-replica
// histograms and the per-window latency bands bin alike.
AF_HD int32_t hist_bin(double lat) {
    const int32_t idx = (int32_t)(d2u(lat) >> (52 - AF_HIST_SUB_BITS)) - ((1023 + AF_HIST_MIN_EXP) << AF_HIST_SUB_BITS);
    return idx < 0 ? 0 : (idx >= AF_HIST_BINS ? AF_HIST_BINS - 1 : idx);
}

// The distribution bands' bin of a gauge value (DESIGN.md §3.7): one bin per value below 64, then 16 log-linear bins per
// octave (a bin is at most 1/16 of its lower edge wide).  results.gauge_bin_edges restates the edges in Python.
AF_HD uint32_t gauge_bin(uint32_t v) {
    if (v < 64u) return v;
#if defined(__CUDA_ARCH__)
    const uint32_t m = 31u - (uint32_t)__clz((int)v);
#else
    const uint32_t m = 31u - (uint32_t)__builtin_clz(v);
#endif
    return 64u + 16u * (m - 6u) + ((v >> (m - 4u)) & 15u);
}

// A latency in 32.32 fixed point: round-to-nearest-even(lat * 2^32) (the scaling by 2^32 is exact).  Per-window latency
// bands add these as two u64 words, so their sums are exact in whatever order the additions land.  A window of a
// group's latency bands is LAT_ROW words: AF_HIST_BINS bin counts, the sum's high word (u >> 32), its low word.
constexpr uint64_t LAT_ROW = AF_HIST_BINS + 2;
AF_HD uint64_t lat_fixed32(double lat) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double2ull_rn(lat * 4294967296.0);
#else
    return (uint64_t)nearbyint(lat * 4294967296.0);       // default rounding mode: to nearest, ties to even
#endif
}

// Occupancy integrals (DESIGN.md §3.8): the time left to the horizon, rest = H - now >= 0, in fixed point with f fraction
// bits, round-to-nearest-even(rest * 2^f), scale = 2^f (the scaling is exact).  A count that changes by delta at now adds
// delta * occ_fixed(H - now) to its column: the column ends as the integral of the count over [0, H) in u64.
AF_HD uint64_t occ_fixed(double rest, double scale) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double2ull_rn(rest * scale);
#else
    return (uint64_t)nearbyint(rest * scale);
#endif
}

// ln(x), finite normal x > 0 (fdlibm e_log.c scheme; see oracle/afrng.py:af_log)
AF_HD_NOINLINE double af_log(double x) {
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10,
                 Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01,
                 Lg3 = 2.857142874366239149e-01, Lg4 = 2.222219843214978396e-01,
                 Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
                 Lg7 = 1.479819860511658591e-01;
    uint64_t b = d2u(x);
    int32_t hx = (int32_t)(b >> 32);
    int32_t k = (hx >> 20) - 1023;
    hx &= 0x000FFFFF;
    int32_t i = (hx + 0x95F64) & 0x100000;
    b = ((uint64_t)(uint32_t)(hx | (i ^ 0x3FF00000)) << 32) | (b & 0xFFFFFFFFull);
    k += i >> 20;
    double f = u2d(b) - 1.0;
    double dk = (double)k;
    double s = af_div(f, 2.0 + f);
    double z = s * s;
    double w = z * z;
    double t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
    double t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
    double r = t2 + t1;
    double hfsq = 0.5 * f * f;
    return dk * ln2_hi - ((hfsq - (s * (hfsq + r) + dk * ln2_lo)) - f);
}

// exp(x) for every double (fdlibm e_exp.c scheme; see oracle/afrng.py:af_exp): +inf above EXP_OVERFLOW, +0.0 below
// EXP_UNDERFLOW, NaN for NaN; the range is settled before the float -> int conversion, which is only defined in range
constexpr double EXP_OVERFLOW = 7.09782712893383973096e+02, EXP_UNDERFLOW = -7.45133219101941108420e+02;
AF_HD double af_exp(double x) {
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10,
                 invln2 = 1.44269504088896338700e+00, P1 = 1.66666666666666019037e-01,
                 P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
    if (x != x) return x;
    if (x > EXP_OVERFLOW) return u2d(0x7FF0000000000000ull);
    if (x < EXP_UNDERFLOW) return 0.0;
    int32_t k = (x >= 0.0) ? (int32_t)(invln2 * x + 0.5) : (int32_t)(invln2 * x - 0.5);
    double dk = (double)k;
    double hi = x - dk * ln2_hi;
    double lo = dk * ln2_lo;
    double r = hi - lo;
    double t = r * r;
    double c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
    double y = 1.0 - ((lo - af_div(r * c, 2.0 - c)) - hi);
    // y * 2^k, y in [0.70, 1.42): through the exponent field while the result is normal; 2^1024 in two steps, and a
    // subnormal result as y * 2^(k+1000) * 2^-1000 (exact, then one rounding)
    if (k >= -1021) {
        if (k == 1024) return u2d(d2u(y) + ((uint64_t)1023 << 52)) * 2.0;
        return u2d(d2u(y) + ((uint64_t)(int64_t)k << 52));
    }
    return u2d(d2u(y) + ((uint64_t)(int64_t)(k + 1000) << 52)) * 9.33263618503218878990e-302;   // 2^-1000
}

// The block number's bits in counter word 1 of a request draw: bits 0-7 hold b & 0xFF (so blocks 0-255 keep the
// counters they always had), bits 26-31 hold b >> 8 -- above the purpose, which takes bits 24-25 (0, 1, 2).  A draw
// has 2^14 distinct blocks; the purpose bits never change, so no request block meets a GEN or SERVER counter.
constexpr uint32_t REQUEST_BLOCKS = 1u << 14;
AF_HD uint32_t block_bits(uint32_t b) { return (b & 0xFFu) | ((b >> 8) << 26); }
// The largest Poisson mean an edge may have: a draw of mean <= 30000 needs more than REQUEST_BLOCKS blocks with
// probability < 1e-50 (DESIGN.md, "AF-RNG"); afh::validate and the sweep check refuse a larger one.
constexpr double EDGE_POISSON_MEAN_MAX = 30000.0;

// One source of uniforms for ONE variate draw (see oracle/afrng.py UniformSource).
struct Src {
    uint32_t k0, k1;      // key = seed
    uint32_t c2, c3;      // replica
    uint32_t idx;         // request id (request draws)
    uint32_t tag;         // purpose<<24 | hop<<8
    uint32_t pos;         // GEN: index of next uniform; request: next half-block
    uint32_t cached;      // block number held in w
    bool is_gen;
    bool have;
    U4 w;

    AF_HD void load(uint32_t b) {
        if (have && cached == b) return;
        U4 c;
        if (is_gen) { c.x = b; c.y = P_GEN << 24; }
        else { c.x = idx; c.y = tag | block_bits(b); }
        c.z = c2; c.w = c3;
        w = philox4x32_10(c, k0, k1);
        cached = b; have = true;
    }
    AF_HD uint32_t word(uint32_t i) const {
        return i == 0 ? w.x : (i == 1 ? w.y : (i == 2 ? w.z : w.w));
    }
    AF_HD double next53() {
        uint32_t p = pos;
        if (is_gen) {
            pos = p + 1;
            load(p >> 1);
            return (p & 1u) ? u53(w.z, w.w) : u53(w.x, w.y);
        }
        pos = p + 2;
        load(p >> 2);
        return (p & 2u) ? u53(w.z, w.w) : u53(w.x, w.y);
    }
    AF_HD void pair32(double& v1, double& v2) {
        if (is_gen) {
            double a = next53(), b = next53();
            v1 = 2.0 * a - 1.0; v2 = 2.0 * b - 1.0;
            return;
        }
        uint32_t p = pos;
        pos = p + 2;
        load(p >> 2);
        if (p & 2u) { v1 = s32(w.z); v2 = s32(w.w); }
        else { v1 = s32(w.x); v2 = s32(w.y); }
    }
};

AF_HD Src make_gen(uint64_t seed, uint64_t replica, uint32_t pos) {
    Src s;
    s.k0 = (uint32_t)seed; s.k1 = (uint32_t)(seed >> 32);
    s.c2 = (uint32_t)replica; s.c3 = (uint32_t)(replica >> 32);
    s.idx = 0; s.tag = 0; s.pos = pos; s.cached = 0; s.is_gen = true; s.have = false;
    s.w = U4{0, 0, 0, 0};
    return s;
}
AF_HD Src make_request(uint64_t seed, uint64_t replica, uint32_t purpose, uint32_t rid, uint32_t hop) {
    Src s;
    s.k0 = (uint32_t)seed; s.k1 = (uint32_t)(seed >> 32);
    s.c2 = (uint32_t)replica; s.c3 = (uint32_t)(replica >> 32);
    s.idx = rid; s.tag = (purpose << 24) | ((hop & 0xFFFFu) << 8);
    s.pos = 2; s.cached = 0; s.is_gen = false; s.have = false;
    s.w = U4{0, 0, 0, 0};
    return s;
}

AF_HD double std_normal(Src& s) {
    for (;;) {
        double v1, v2;
        s.pair32(v1, v2);
        double q = v1 * v1 + v2 * v2;
        if (q > 0.0 && q < 1.0) return v1 * af_sqrt(af_div(-2.0 * af_log(q), q));
    }
}

AF_HD int64_t poisson(double lam, Src& s) {
    int64_t n = 0;
    double rem = lam;
    while (rem > 0.0) {
        double c = rem < 256.0 ? rem : 256.0;
        rem = rem - c;
        double limit = af_exp(-c);
        double p = 1.0;
        for (;;) {
            p = p * (1.0 - s.next53());
            if (p <= limit) break;
            ++n;
        }
    }
    return n;
}

// general_sampler, reference samplers/common_helpers.py:49-89
AF_HD double sample_rv(int dist, double mean, double sigma, Src& s) {
    if (dist == 3 /*EXPONENTIAL*/) return mean * -af_log(1.0 - s.next53());
    if (dist == 1 /*NORMAL*/) { double v = mean + sigma * std_normal(s); return v > 0.0 ? v : 0.0; }
    if (dist == 2 /*LOG_NORMAL*/) return af_exp(mean + sigma * std_normal(s));
    if (dist == 4 /*UNIFORM*/) return s.next53();
    return (double)poisson(mean, s);  /* POISSON */
}

// One edge traversal's random numbers (reference runtime/actors/edge.py:78,90): the dropout
// uniform and -- unless the request is dropped -- the latency variate.  Deliberately NOT
// inlined: the engine sends requests from five places and the variate code is the bulk of the
// kernel's instructions; one shared body keeps the hot loop inside the instruction cache.
struct EdgeDraw { double u; double transit; };
AF_HD_NOINLINE EdgeDraw edge_draw(uint64_t seed, uint64_t replica, uint32_t rid, uint32_t hop, int dist,
                                  double mean, double sigma, double dropout) {
    Src s = make_request(seed, replica, P_EDGE, rid, hop);
    s.load(0);
    EdgeDraw d;
    d.u = u53(s.w.x, s.w.y);
    d.transit = 0.0;
    if (!(d.u < dropout)) d.transit = sample_rv(dist, mean, sigma, s);
    return d;
}

// The generator's draws (samplers/poisson_poisson.py:58-71, gaussian_poisson.py:70-83); `pos`
// is the index of the next uniform of the replica's sequential GEN stream.
struct GenDraw { double value; uint32_t pos; };
AF_HD_NOINLINE GenDraw gen_users(uint64_t seed, uint64_t replica, uint32_t pos, int users_dist, double mean,
                                 double sigma) {
    Src s = make_gen(seed, replica, pos);
    GenDraw g;
    if (users_dist == 1 /*NORMAL*/) {
        double v = mean + sigma * std_normal(s);
        g.value = v > 0.0 ? v : 0.0;        // truncated_gaussian_generator
    } else {
        g.value = (double)poisson(mean, s);
    }
    g.pos = s.pos;
    return g;
}

}  // namespace afr
