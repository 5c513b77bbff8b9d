// lora_common.cuh -- small host/device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define LB_HD __host__ __device__ __forceinline__
#define LB_D __device__ __forceinline__
#else
#define LB_HD inline
#define LB_D inline
#endif

namespace lb {

// The largest float below the double M_PI (0x40490FDA; the next float, 0x40490FDB, is above it).  The reference unwraps phase
// differences with "while ((phase2 - phase) > M_PI)" (lib/decoder_impl.cc:236-237): a float difference promoted to double.
// For a float d, (double)d > M_PI  <=>  d > LB_PI_BELOW, and (double)d < -M_PI  <=>  d < -LB_PI_BELOW, exactly -- the test
// needs no fp64 conversion / compare per sample (they were 15 % of the stream kernel's stall samples).
#define LB_PI_BELOW 3.14159250259399414f

// ---- complex arithmetic ---------------------------------------------------------------------
// On the device a complex value can be handled as a 64-bit register pair (lb_u64).  The pair operations below are two
// scalar fp32 operations with explicit round-to-nearest (Hopper has no packed fp32 instructions): the explicit rounding
// keeps ptxas from contracting a product and a sum into one FFMA, so every kernel rounds exactly where its source says.
// LB_PACKED_CMUL selects the product form cmul(a, b) = fma(b, a.x, (-b.y, b.x) * a.y) for the translation units that
// use it; the host build (CPU emulation of the kernels for the non-GPU tests) uses the plain scalar formulas.
typedef unsigned long long lb_u64;
#ifdef __CUDA_ARCH__
LB_D lb_u64 pk2(float lo, float hi) { lb_u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
LB_D float2 up2(lb_u64 v) { float2 r; asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v)); return r; }
LB_D lb_u64 add2(lb_u64 a, lb_u64 b) { const float2 x = up2(a), y = up2(b); return pk2(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y)); }
LB_D lb_u64 sub2(lb_u64 a, lb_u64 b) { const float2 x = up2(a), y = up2(b); return pk2(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y)); }
LB_D lb_u64 mul2(lb_u64 a, lb_u64 b) { const float2 x = up2(a), y = up2(b); return pk2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y)); }
LB_D lb_u64 fma2(lb_u64 a, lb_u64 b, lb_u64 c) {
    const float2 x = up2(a), y = up2(b), z = up2(c);
    return pk2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
LB_D float2 cadd(float2 a, float2 b) { return up2(add2(pk2(a.x, a.y), pk2(b.x, b.y))); }
LB_D float2 csub(float2 a, float2 b) { return up2(sub2(pk2(a.x, a.y), pk2(b.x, b.y))); }
// packed product with a compile-time constant (used inside the radix butterflies)
LB_D float2 cmul_const(float2 a, float wx, float wy) {
    return up2(fma2(pk2(wx, wy), pk2(a.x, a.x), mul2(pk2(-wy, wx), pk2(a.y, a.y))));
}
#ifdef LB_PACKED_CMUL
// plain complex product (the reference multiplies by the down-chirp, not its conjugate,
// lib/decoder_impl.cc:436-438):  a*b = (b.x, b.y)*a.x + (-b.y, b.x)*a.y
LB_D float2 cmul(float2 a, float2 b) {
    return up2(fma2(pk2(b.x, b.y), pk2(a.x, a.x), mul2(pk2(-b.y, b.x), pk2(a.y, a.y))));
}
// a * w + c
LB_D float2 cfma(float2 a, float2 w, float2 c) {
    return up2(fma2(pk2(w.x, w.y), pk2(a.x, a.x), fma2(pk2(-w.y, w.x), pk2(a.y, a.y), pk2(c.x, c.y))));
}
LB_D float cnorm2(float2 a) { const float2 q = up2(mul2(pk2(a.x, a.y), pk2(a.x, a.y))); return q.x + q.y; }
#endif
#else
LB_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
LB_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
#endif
#if !defined(__CUDA_ARCH__) || !defined(LB_PACKED_CMUL)
LB_HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
LB_HD float2 cfma(float2 a, float2 w, float2 c) {
    return make_float2(fmaf(a.x, w.x, fmaf(-a.y, w.y, c.x)), fmaf(a.x, w.y, fmaf(a.y, w.x, c.y)));
}
LB_HD float cnorm2(float2 a) { return fmaf(a.x, a.x, a.y * a.y); }
#endif
LB_HD float2 cconj(float2 a) { return make_float2(a.x, -a.y); }

// cos/sin(2*pi*e/32), e = 0..15, as literals so that they fold after unrolling
LB_HD float cos32(int e) {
    switch (e & 15) {
    case 0: return 1.0f;
    case 1: return 0.98078528040323043f;
    case 2: return 0.92387953251128674f;
    case 3: return 0.83146961230254524f;
    case 4: return 0.70710678118654757f;
    case 5: return 0.55557023301960229f;
    case 6: return 0.38268343236508984f;
    case 7: return 0.19509032201612833f;
    case 8: return 0.0f;
    case 9: return -0.19509032201612833f;
    case 10: return -0.38268343236508984f;
    case 11: return -0.55557023301960229f;
    case 12: return -0.70710678118654757f;
    case 13: return -0.83146961230254524f;
    case 14: return -0.92387953251128674f;
    default: return -0.98078528040323043f;
    }
}
// sin(2*pi*e/32) = cos(2*pi*|e-8|/32) for e in [0,16)
LB_HD float sin32(int e) { return cos32(e > 8 ? e - 8 : 8 - e); }

// multiply by W_32^e = exp(-2*pi*i*e/32), e in [0,16), e known at compile time after unrolling
LB_HD float2 mul_w32(float2 a, int e) {
#ifdef __CUDA_ARCH__
    if (e == 0) return a;
    if (e == 8) return up2(mul2(pk2(a.y, a.x), pk2(1.0f, -1.0f)));          // * (-i): swap + one sign
    return cmul_const(a, cos32(e), -sin32(e));                               // W = c - i s
#else
    const float h = 0.70710678118654757f;
    switch (e) {
    case 0: return a;
    case 8: return make_float2(a.y, -a.x);                       // * (-i)
    case 4: return make_float2((a.x + a.y) * h, (a.y - a.x) * h);    // * (1 - i)/sqrt2
    case 12: return make_float2((a.y - a.x) * h, -(a.x + a.y) * h);  // * (-1 - i)/sqrt2
    default: {
        const float c = cos32(e);
        const float s = sin32(e);
        // W = c - i s  ->  (a.x + i a.y)(c - i s) = (a.x c + a.y s) + i (a.y c - a.x s)
        return make_float2(fmaf(a.x, c, a.y * s), fmaf(a.y, c, -a.x * s));
    }
    }
#endif
}

// in-register radix-2 DIF DFT of R points (forward, e^{-j}); X[k] ends up at v[bitrev(k)]
template <int R>
LB_HD void dft_dif(float2 *v) {
#pragma unroll
    for (int len = R; len >= 2; len >>= 1) {
        const int half = len >> 1;
#pragma unroll
        for (int g0 = 0; g0 < R; g0 += len) {
#pragma unroll
            for (int k = 0; k < half; k++) {
                const float2 a = v[g0 + k], b = v[g0 + k + half];
                v[g0 + k] = cadd(a, b);
                v[g0 + k + half] = mul_w32(csub(a, b), k * (32 / len));
            }
        }
    }
}

template <int R>
LB_HD constexpr int bitrev(int k) {
    int r = 0;
    for (int b = 1, t = R >> 1; b < R; b <<= 1, t >>= 1)
        if (k & b) r |= t;
    return r;
}

// argmax key: larger |.|^2 wins, ties go to the smaller index (std::max_element keeps the
// first maximum, lib/decoder_impl.cc:463).  mag2 >= 0 so its bit pattern is monotonic.
LB_HD unsigned long long pack_key(float mag2, uint32_t idx) {
    union { float f; uint32_t u; } c;
    c.f = mag2;
    return ((unsigned long long)c.u << 32) | (unsigned long long)(0xFFFFFFFFu - idx);
}
LB_HD uint32_t key_idx(unsigned long long k) { return 0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull); }
LB_HD float key_mag2(unsigned long long k) {
    union { float f; uint32_t u; } c;
    c.u = (uint32_t)(k >> 32);
    return c.f;
}
#ifdef __CUDACC__
// arg(x + i y) for the instantaneous-frequency passes (the reference's std::arg, lib/decoder_impl.cc:232-233, one per sample).
// CUDA's atan2f is a rational approximation with two divisions and their slow-path checks: 65 instructions, 22 % of the
// stream kernel's instructions.  This one: one IEEE division, t + t s P(s) with s = t^2 and a
// degree-7 minimax P fitted to relative error (1.7e-8 before rounding), then the octant fix-ups: 26 instructions, measured
// max error 1.8 ulp on 4e6 random points (CUDA documents 2 ulp for atan2f, so the two are interchangeable for parity:
// both differ from glibc's result in the last bit on a fraction of the samples).  Zero, infinite and NaN inputs follow C99.
LB_HD float lb_atan2f(float y, float x) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
#ifdef __CUDA_ARCH__
    float q = __fdiv_rn(mn, mx);
    const float inf = __int_as_float(0x7f800000);
    const bool x_neg = __float_as_int(x) < 0;
#else                                                                    // the host build (tests/test_host_emulation.py): IEEE division as well
    float q = mn / mx;
    const float inf = INFINITY;
    const bool x_neg = signbit(x);
#endif
    if (mx == 0.0f) q = 0.0f;                                            // atan2(+-0, +-0)
    if (mx == inf) q = mn == mx ? 1.0f : 0.0f;                           // infinite operands
    const float s = q * q;
    float p = 0.0029206566978245974f;
    p = fmaf(p, s, -0.01636778749525547f);
    p = fmaf(p, s, 0.04321163520216942f);
    p = fmaf(p, s, -0.07552195340394974f);
    p = fmaf(p, s, 0.10665995627641678f);
    p = fmaf(p, s, -0.14211052656173706f);
    p = fmaf(p, s, 0.19993773102760315f);
    p = fmaf(p, s, -0.33333152532577515f);
    float r = fmaf(q * s, p, q);
    if (ay > ax) r = 1.5707963705062866211f - r;
    if (x_neg) r = 3.1415927410125732422f - r;
    const float sum = ax + ay;
    if (sum != sum) return sum;                                          // NaN in, NaN out
    return copysignf(r, y);
}
// Maximum key of the warp in every lane: two REDUX (the high words, then the low words of the lanes that hold the maximal
// high word) instead of five dependent 64-bit shuffle + compare rounds (10 SHFL + 20 ALU; ~6 % of k1_rows<11>'s stall
// samples sat on that chain)
LB_D unsigned long long warp_max_key(unsigned long long k) {
    const uint32_t hi = (uint32_t)(k >> 32);
    const uint32_t m = __reduce_max_sync(0xffffffffu, hi);
    const uint32_t l = __reduce_max_sync(0xffffffffu, hi == m ? (uint32_t)k : 0u);
    return ((unsigned long long)m << 32) | (unsigned long long)l;
}
// Maximum key of each aligned group of W lanes (W a power of two <= 32) in every lane of the group; W = 32 is warp_max_key
template <int W>
LB_D unsigned long long group_max_key(unsigned long long k) {
    if (W == 32) return warp_max_key(k);
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, k, o);
        k = v > k ? v : k;
    }
    return k;
}
#endif

}  // namespace lb
