// rng.cuh - per-trial pseudo-random stream and variate samplers, device side.
//
// Drop-in arithmetic for the reference's cmb_random (src/cmb_random.c,
// include/cmb_random.h): the same generator (sfc64, 256-bit state, seeded by
// four splitmix64 outputs plus 20 discarded draws) and the same McFarland
// ziggurat samplers over the same 256-layer tables, so that a trial seeded with
// cmb_random_fmix64(master, index) consumes and produces the identical stream.
//
// GPU mapping: the four 64-bit state words live in registers (8 x 32-bit) for
// the whole trial; the 2 KB layer-width tables used by 98.4 % of the draws are
// staged once per CTA in shared memory (lanes index them with unrelated
// indices, which constant memory would serialise); the overhang tables used by
// the remaining 1.6 % stay in global memory behind L1/L2.
//
// Bit parity rules (SURVEY.md section 7, "Bit parity of doubles"): every
// floating-point operation is spelled with a round-to-nearest intrinsic so that
// nvcc cannot contract a*b+c into an FMA (the reference build has no FMA), and
// uint64/int64 -> double conversions use the _rn forms (= C casts on x86-64).
#pragma once

#include <cstdint>
#ifndef CMB_HOST_BUILD     // tests/cmb_engine_host.cpp compiles this text for the CPU
#include <cuda_runtime.h>
#endif

#include "glibc_exp.cuh"
#include "zig_tables.cuh"

namespace cimba_b200 {

// ------------------------------------------------------------- host + device
// cmb_random_fmix64, src/cmb_random.c:70-80
__host__ __device__ __forceinline__ uint64_t fmix64(uint64_t seed, uint64_t nonce)
{
    uint64_t h = seed + nonce;
    h ^= h >> 33;
    h *= 0xff51afd7ed558ccdULL;
    h ^= h >> 33;
    h *= 0xc4ceb9fe1a85ec53ULL;
    h ^= h >> 33;
    return h;
}

// Shared-memory staging area for the two hot tables.
struct ZigHot {
    double exp_x[256];
    double nor_x[256];
};

__device__ __forceinline__ void stage_zig_hot(ZigHot &hot, bool want_normal)
{
    for (unsigned i = threadIdx.x; i < 256u; i += blockDim.x) {
        hot.exp_x[i] = zig::zig_exp_x[i];
        hot.nor_x[i] = want_normal ? zig::zig_nor_x[i] : 0.0;
    }
}

// exp() of the ziggurat wedge tests (src/cmb_random.c:255, :345), out of line: reached by 0.04 % of the draws, and
// an inlined copy at each of the four call sites would only cost instruction-cache room
__device__ __noinline__ double zig_exp(double x)
{
    return glibc_exp(x);
}

constexpr double TWO_POW_64 = 18446744073709551616.0;
constexpr double TWO_POW_63 = 9223372036854775808.0;
constexpr double TWO_POW_M53 = 1.1102230246251565404e-16;

// A double converted to an integer as the reference's build converts it.  C leaves (long)x and (unsigned)x undefined when the
// truncated x does not fit (C11 6.3.1.4); gcc on x86-64 emits the 64-bit cvttsd2si for both, which gives the truncated x when
// |x| < 2^63 and 0x8000000000000000 for anything else (NaN included), and (unsigned)x keeps the low 32 bits of that.  The
// device's cvt.rzi instructions saturate instead.  (unsigned)(uint64_t)x86_cvttsd2si(x) is the reference's (unsigned)x.
__host__ __device__ __forceinline__ int64_t x86_cvttsd2si(double x)
{
    return fabs(x) < TWO_POW_63 ? (int64_t)x : INT64_MIN;
}

#ifndef CMB_HOST_BUILD
// Integer multipliers read from the constant bank.  ptxas rewrites a multiply by an immediate 1 or power of two as an add or a
// shift (the half-rate ALU pipe); a constant-bank operand it cannot see into keeps the operation an IMAD (the FMA pipe).
static __constant__ uint32_t imad_k[3] = {1u << 21, 1u << 24, 1u << 11};
#define IMAD_K2P21 imad_k[0]
#define IMAD_K2P24 imad_k[1]
#define IMAD_K2P11 imad_k[2]

__device__ __forceinline__ uint64_t u64_of(uint32_t lo, uint32_t hi)
{
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
    return r;
}

__device__ __forceinline__ void u32_of(uint64_t v, uint32_t &lo, uint32_t &hi)
{
    asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
}

__device__ __forceinline__ uint64_t imad_wide(uint32_t x, uint32_t y, uint64_t z)       // x * y + z, 64-bit
{
    uint64_t r;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(x), "r"(y), "l"(z));
    return r;
}

__device__ __forceinline__ uint32_t imad_lo(uint32_t x, uint32_t y, uint32_t z)         // low word of x * y + z
{
    uint32_t r;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(x), "r"(y), "r"(z));
    return r;
}

__device__ __forceinline__ uint32_t imad_hi(uint32_t x, uint32_t y, uint32_t z)         // high word of x * y, plus z
{
    uint32_t r;
    asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(x), "r"(y), "r"(z));
    return r;
}
#endif

struct Sfc64 {
    uint64_t a, b, c, d;

    // cmb_random_sfc64, src/cmb_random.c:54-62
    __device__ __forceinline__ uint64_t next()
    {
        const uint64_t out = a + b + d++;
        a = b ^ (b >> 11);
#if !defined(SFC64_NO_IMAD) && !defined(CMB_HOST_BUILD)
        // c + (c << 3) = 9 c as IMAD.WIDE + IMAD (FMA pipe) instead of LEA + LEA.HI.X (the half-rate ALU pipe, the busiest pipe of
        // every event loop here).  Same value, bit for bit.
        // (ptxas turns a multiply-add by 1 back into IADD3, so the generator's additions stay where they are.)
        {
            uint32_t lo, hi;
            asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(c));
            uint64_t w;
            asm("mul.wide.u32 %0, %1, 9;" : "=l"(w) : "r"(lo));
            uint32_t wl, wh;
            asm("mov.b64 {%0, %1}, %2;" : "=r"(wl), "=r"(wh) : "l"(w));
            asm("mad.lo.u32 %0, %1, 9, %2;" : "=r"(wh) : "r"(hi), "r"(wh));
            asm("mov.b64 %0, {%1, %2};" : "=l"(b) : "r"(wl), "r"(wh));
        }
#else
        b = c + (c << 3);
#endif
        c = ((c << 24) | (c >> 40)) + out;
        return out;
    }

    // The same step as next() with its shifts also on the FMA pipe, for a kernel whose ALU pipe is the busier one
    // (mm1_kernel).  It is not the default: in the G/G/1 and M/M/c kernels and the static tier it measured slower on the H100.
    __device__ __forceinline__ uint64_t next_imad()
    {
#if !defined(SFC64_NO_IMAD) && !defined(CMB_HOST_BUILD)
        // The shifts run as IMAD on the FMA pipe instead of SHF on the half-rate ALU pipe, the busiest pipe of every event loop
        // here; the additions and XORs stay on the ALU pipe as three-input IADD3 / LOP3.  Integer arithmetic is exact: the
        // same values, bit for bit (define SFC64_NO_IMAD for the plain form).
        //   b ^ (b >> 11)      = {b.lo ^ hi(b.lo * 2^21) ^ lo(b.hi * 2^21), b.hi ^ hi(b.hi * 2^21)}
        //   c + (c << 3) = 9 c = c.lo * 9 (wide), + c.hi * 9 in the high word
        //   rotl(c, 24)        = c.lo * 2^24 (wide) + {hi(c.hi * 2^24), lo(c.hi * 2^24)}   (no two terms share a bit)
        const uint64_t out = a + b + d++;
        uint32_t bl, bh, cl, ch;
        u32_of(b, bl, bh);
        u32_of(c, cl, ch);
        {
            uint32_t wl, wh;
            u32_of(imad_wide(bh, IMAD_K2P21, 0ull), wl, wh);
            a = u64_of(bl ^ imad_hi(bl, IMAD_K2P21, 0u) ^ wl, bh ^ wh);
        }
        {
            uint32_t wl, wh;
            u32_of(imad_wide(cl, 9u, 0ull), wl, wh);
            b = u64_of(wl, imad_lo(ch, 9u, wh));
        }
        {
            uint32_t wl, wh;
            u32_of(imad_wide(ch, IMAD_K2P24, 0ull), wl, wh);
            c = imad_wide(cl, IMAD_K2P24, 0ull) + u64_of(wh, wl) + out;
        }
        return out;
#else
        return next();
#endif
    }

    // The inverse of next(): puts the last output back.  sfc64's state transition is a bijection
    // (a' = b ^ (b >> 11), b' = 9c, c' = rotl(c, 24) + out, d' = d + 1), so a kernel that runs a few
    // raw draws ahead of the simulation can hand the stream back to the reference-order slow path.
    __device__ __forceinline__ void rewind()
    {
        const uint64_t pc = b * 0x8e38e38e38e38e39ULL;  // 9^-1 mod 2^64
        uint64_t pb = a;                                // undo b ^ (b >> 11)
        pb ^= pb >> 11;
        pb ^= pb >> 22;
        pb ^= pb >> 44;
        const uint64_t out = c - ((pc << 24) | (pc >> 40));
        d -= 1u;
        a = out - pb - d;
        b = pb;
        c = pc;
    }

    // cmb_random_initialize, src/cmb_random.c:112-124 (splitmix64 at :99-106)
    __device__ __forceinline__ void seed(uint64_t s)
    {
        uint64_t w[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint64_t z = (s += 0x9e3779b97f4a7c15ULL);
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
            w[i] = z ^ (z >> 31);
        }
        a = w[0];
        b = w[1];
        c = w[2];
        d = w[3];
#pragma unroll 1
        for (int i = 0; i < 20; i++) {
            (void)next();
        }
    }

    // cmb_random(), include/cmb_random.h:149-152
    __device__ __forceinline__ double uniform01()
    {
        return __dmul_rn(__ull2double_rn(next() >> 11), TWO_POW_M53);
    }

    // cmb_random_uniform, include/cmb_random.h:165-173
    __device__ __forceinline__ double uniform(double lo, double hi)
    {
        return __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), uniform01()));
    }

    // cmb_random_bernoulli, include/cmb_random.h:749-754
    __device__ __forceinline__ unsigned bernoulli(double p)
    {
        return uniform01() <= p ? 1u : 0u;
    }

    // cmb_random_dice, include/cmb_random.h:840-846.  lo + x can round up to 2^63 when hi is near INT64_MAX: the reference's
    // (long) conversion then gives INT64_MIN, which x86_cvttsd2si states.
    __device__ __forceinline__ long long dice(long long lo, long long hi)
    {
        const double x = __dmul_rn(__ll2double_rn(hi - lo + 1), uniform01());
        return x86_cvttsd2si(floor(__dadd_rn(__ll2double_rn(lo), x)));
    }

    // ------------------------------------------------------------ exponential

    // Is u inside the rectangular body of the exponential ziggurat?
    static __device__ __forceinline__ bool exp_is_hot(uint64_t u)
    {
        return (unsigned)(u & 0xffu) <= ZIG_EXP_MAX;
    }

    // include/cmb_random.h:321-325: width of layer (u & 255) times the FULL u
    static __device__ __forceinline__ double exp_hot(const ZigHot &hot, uint64_t u)
    {
        return __dmul_rn(hot.exp_x[u & 0xffu], __ull2double_rn(u));
    }

    // cmi_random_exp_not_hot, src/cmb_random.c:216-285
    __device__ __forceinline__ double exp_cold(uint64_t ux)
    {
        double shift = 0.0;
        for (;;) {
            uint64_t uy = next();
            unsigned j = (unsigned)(uy & 0xffu);
            if (next() >= zig::zig_exp_prob[j]) {
                j = zig::zig_exp_alias[j];
            }
            if (j > 0u) {
                const double xj = zig::zig_exp_x[j];
                const double dx = __dsub_rn(zig::zig_exp_x[j - 1u], xj);
                for (;;) {
                    if (uy > (UINT64_MAX - ux)) {
                        uy = UINT64_MAX - uy;
                        ux = UINT64_MAX - ux;
                    }
                    const uint64_t gap = (UINT64_MAX - ux) - uy;
                    // zig_exp_convert_x, src/cmb_random.c:198-201
                    const double x = __dadd_rn(__dmul_rn(xj, TWO_POW_64),
                                               __dmul_rn(dx, __ull2double_rn(ux)));
                    if (gap >= zig::zig_exp_concavity[j]) {
                        return __dadd_rn(x, shift);
                    }
                    // zig_exp_convert_y, src/cmb_random.c:203-206
                    const double y0 = zig::zig_exp_y[j - 1u];
                    const double y = __dadd_rn(__dmul_rn(y0, TWO_POW_64),
                                               __dmul_rn(__dsub_rn(zig::zig_exp_y[j], y0),
                                                         __ull2double_rn(uy)));
                    if (y <= zig_exp(-x)) {          // src/cmb_random.c:255: glibc's exp, bit for bit (glibc_exp.cuh)
                        return __dadd_rn(x, shift);
                    }
                    uy = next();
                    ux = next();
                }
            }
            shift = __dadd_rn(shift, ZIG_EXP_TAIL);
            ux = next();
            const unsigned i = (unsigned)(ux & 0xffu);
            if (i <= ZIG_EXP_MAX) {
                return __dadd_rn(__dmul_rn(zig::zig_exp_x[i], __ull2double_rn(ux)), shift);
            }
        }
    }

    // cmb_random_std_exponential, include/cmb_random.h:319-329
    __device__ __forceinline__ double std_exponential(const ZigHot &hot)
    {
        const uint64_t u = next();
        return exp_is_hot(u) ? exp_hot(hot, u) : exp_cold(u);
    }

    // the same draw with the layer table read from global memory (L1-resident): for
    // kernels that cannot spare shared memory for the table
    __device__ __forceinline__ double std_exponential_global()
    {
        const uint64_t u = next();
        return exp_is_hot(u) ? __dmul_rn(zig::zig_exp_x[u & 0xffu], __ull2double_rn(u)) : exp_cold(u);
    }

    // cmb_random_exponential, include/cmb_random.h:344-352
    __device__ __forceinline__ double exponential(const ZigHot &hot, double mean)
    {
        return __dmul_rn(mean, std_exponential(hot));
    }

    // cmb_random_erlang, include/cmb_random.h:366-378
    __device__ __forceinline__ double erlang(const ZigHot &hot, unsigned k, double m)
    {
        double x = 0.0;
        for (unsigned i = 0u; i < k; i++) {
            x = __dadd_rn(x, exponential(hot, m));
        }
        return x;
    }

    // ----------------------------------------------------------------- normal

    __device__ __forceinline__ int64_t draw63()         // zig_sample63, src/cmb_random.c:333-337
    {
        return (int64_t)(next() & (uint64_t)INT64_MAX);
    }

    static __device__ __forceinline__ double nor_x_of(unsigned j, int64_t ix)
    {                                                   // zig_nor_convert_x, :321-324
        const double xj = zig::zig_nor_x[j];
        return __dadd_rn(__dmul_rn(xj, TWO_POW_63),
                         __dmul_rn(__dsub_rn(zig::zig_nor_x[j - 1u], xj), __ll2double_rn(ix)));
    }

    static __device__ __forceinline__ double nor_y_of(unsigned j, int64_t iy)
    {                                                   // zig_nor_convert_y, :326-329
        const double y0 = zig::zig_nor_y[j - 1u];
        return __dadd_rn(__dmul_rn(y0, TWO_POW_63),
                         __dmul_rn(__dsub_rn(zig::zig_nor_y[j], y0),
                                   __ull2double_rn((uint64_t)iy)));
    }

    static __device__ __forceinline__ double nor_pdf_scaled(double x)
    {                                                   // sc_nor_pdf, :340-343
        return zig_exp(__dmul_rn(__dmul_rn(-0.5, x), x));    // glibc's exp, bit for bit (glibc_exp.cuh)
    }

    // cmi_random_nor_not_hot, src/cmb_random.c:352-451
    __device__ __forceinline__ double nor_cold(const ZigHot &hot, int64_t ix)
    {
        const double sign = (ix < 0) ? -1.0 : 1.0;
        ix &= INT64_MAX;
        int64_t iy = draw63();
        unsigned j = (unsigned)(iy & 0xff);
        if (ix >= zig::zig_nor_prob[j]) {
            j = zig::zig_nor_alias[j];
        }
        if (j > ZIG_NOR_INFLECTION) {
            for (;;) {
                const double x = nor_x_of(j, ix);
                const int64_t gap = (INT64_MAX - ix) - iy;
                if (gap >= 0) {
                    return __dmul_rn(sign, x);
                }
                if (gap + zig::zig_nor_convexity[j] >= 0) {
                    if (nor_y_of(j, iy) < nor_pdf_scaled(x)) {
                        return __dmul_rn(sign, x);
                    }
                }
                ix = draw63();
                iy = draw63();
            }
        }
        else if (j == 0u) {
            double x, z;
            do {
                x = __dmul_rn(ZIG_NOR_INV_TAIL, exponential(hot, 1.0));
                z = exponential(hot, 1.0);
            } while (__dmul_rn(2.0, z) <= __dmul_rn(x, x));
            return __dmul_rn(sign, __dadd_rn(x, ZIG_NOR_TAIL));
        }
        else if (j < ZIG_NOR_INFLECTION) {
            for (;;) {
                if (iy > INT64_MAX - ix) {
                    iy = INT64_MAX - iy;
                    ix = INT64_MAX - ix;
                }
                const double x = nor_x_of(j, ix);
                const int64_t gap = (INT64_MAX - ix) - iy;
                if (gap >= zig::zig_nor_concavity[j]) {
                    return __dmul_rn(sign, x);
                }
                if (nor_y_of(j, iy) <= nor_pdf_scaled(x)) {
                    return __dmul_rn(sign, x);
                }
                ix = draw63();
                iy = draw63();
            }
        }
        else {
            for (;;) {
                const double x = nor_x_of(j, ix);
                const int64_t gap = (INT64_MAX - ix) - iy;
                if (gap >= zig::zig_nor_concavity[j]) {
                    return __dmul_rn(sign, x);
                }
                if (gap + zig::zig_nor_convexity[j] > 0) {
                    if (nor_y_of(j, iy) < nor_pdf_scaled(x)) {
                        return __dmul_rn(sign, x);
                    }
                }
                ix = draw63();
                iy = draw63();
            }
        }
    }

    // cmb_random_std_normal, include/cmb_random.h:206-215
    __device__ __forceinline__ double std_normal(const ZigHot &hot)
    {
        const int64_t ix = (int64_t)next();
        const unsigned i = (unsigned)(ix & 0xff);
        return (i <= ZIG_NOR_MAX) ? __dmul_rn(hot.nor_x[i], __ll2double_rn(ix))
                                  : nor_cold(hot, ix);
    }

    // cmb_random_normal, include/cmb_random.h:230-235
    __device__ __forceinline__ double normal(const ZigHot &hot, double mu, double sigma)
    {
        return __dadd_rn(mu, __dmul_rn(sigma, std_normal(hot)));
    }
};

}  // namespace cimba_b200
