// Shared device helpers for the FAcodec sm_90a hot path.
// Activations are CHANNELS-LAST fp32: a tensor the reference calls [B, C, T] lives in HBM as
// [B][T][C] ("frames x channels").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fac {

// ---- reflect / zero padding index map --------------------------------------------------
// Restates encodec.py:96-113 (pad1d) for one padded position p in [-pad_left, L + pad_right):
// reflect mode with the short-input branch (x zero-extended to length max_pad+1 before the
// reflection, then truncated).  Returns the source row, or -1 when the padded value is 0.
struct PadMap {
    int L;        // valid input length (rows)
    int Le;       // L, or max_pad + 1 when L <= max_pad (reflect mode)
    int reflect;  // 1 = reflect, 0 = zero pad
    __host__ __device__ static PadMap make(int L, int pad_left, int pad_right, int reflect) {
        PadMap m;
        m.L = L;
        m.reflect = reflect;
        int mp = pad_left > pad_right ? pad_left : pad_right;
        m.Le = (reflect && L <= mp) ? mp + 1 : L;
        return m;
    }
    // Lane b of a batch whose lanes have their own lengths (lane_len [B], null: every lane has Tin rows): the map of the
    // lane's own sequence, so no padded position reads a row at or past the lane's end.
    __host__ __device__ static PadMap lane(const int* lane_len, int b, int Tin, int pad_left, int pad_right, int reflect) {
        return make(lane_len ? lane_len[b] : Tin, pad_left, pad_right, reflect);
    }
    __host__ __device__ __forceinline__ int src(int p) const {
        if (p >= 0 && p < L) return p;
        if (!reflect) return -1;
        int q = p < 0 ? -p : (p < Le ? p : 2 * Le - 2 - p);
        return (q >= 0 && q < L) ? q : -1;
    }
};

// ---- Snake activation, dac/nn/layers.py:17-24 -------------------------------------------
// x + (alpha + 1e-9)^-1 * sin(alpha x)^2 ; inv_alpha is precomputed on the host in fp32.
__device__ __forceinline__ float snake_f(float x, float alpha, float inv_alpha) {
    float s = sinf(alpha * x);
    return x + inv_alpha * (s * s);
}

// sin(x)^2 without quadrant logic: sin^2 is pi-periodic, so reduce x mod pi (two-constant
// Cody-Waite, exact for |k| < 2^12) to r in [-pi/2, pi/2] and evaluate the odd Taylor
// polynomial up to r^13 (truncation < 1e-9).  Measured vs fp64: max |err| 2e-7, rms 4e-8 (sinf^2: 1.2e-7 / 4e-8).  ~15 instructions
// instead of the ~40 + slow path of sinf(); arguments beyond 4096 take the sinf() path.
static __device__ __noinline__ float sin2_slow(float x) {
    float s = sinf(x);
    return s * s;
}
// INLINE_SLOW: kernels that re-allocate registers with setmaxnreg must not contain ABI calls (ptxas 12.9
// crashes on the combination), so they inline the rarely-taken sinf() path instead of calling it.
// polynomial path only: |x| <= 4096 (callers check)
__device__ __forceinline__ float sin2_poly(float x) {
    float k = rintf(x * 0.318309886183790672f);
    float r = fmaf(k, -3.14159274101257324f, x);      // pi_hi (fp32)
    r = fmaf(k, 8.74227765734758578e-8f, r);          // -pi_lo: pi = pi_hi + pi_lo, pi_lo = -8.742e-8
    float r2 = r * r;
    float p = fmaf(r2, 1.60590438368216146e-10f, -2.50521083854417188e-8f);
    p = fmaf(p, r2, 2.75573192239858907e-6f);
    p = fmaf(p, r2, -1.98412698412698413e-4f);
    p = fmaf(p, r2, 8.33333333333333333e-3f);
    p = fmaf(p, r2, -1.66666666666666667e-1f);
    p = fmaf(p * r2, r, r);                           // r + r^3 * (...)
    return p * p;
}
template <bool INLINE_SLOW = false>
__device__ __forceinline__ float sin2_f(float x) {
    if (fabsf(x) > 4096.0f) {
        if constexpr (INLINE_SLOW) { float s = sinf(x); return s * s; }
        else return sin2_slow(x);
    }
    return sin2_poly(x);
}
template <bool INLINE_SLOW = false>
__device__ __forceinline__ float snake_fast(float x, float alpha, float inv_alpha) {
    return fmaf(inv_alpha, sin2_f<INLINE_SLOW>(alpha * x), x);
}
// Four channels of one row at once: ONE range check for the four arguments (3 FMNMX + 1 compare instead of four
// compare-and-branch pairs; same arithmetic per element as snake_fast).
template <bool INLINE_SLOW = false>
__device__ __forceinline__ float4 snake4(float4 x, float4 al, float4 ia) {
    const float y0 = al.x * x.x, y1 = al.y * x.y, y2 = al.z * x.z, y3 = al.w * x.w;
    const float m = fmaxf(fmaxf(fabsf(y0), fabsf(y1)), fmaxf(fabsf(y2), fabsf(y3)));
    float4 o;
    if (m > 4096.0f) {
        o.x = fmaf(ia.x, sin2_f<INLINE_SLOW>(y0), x.x); o.y = fmaf(ia.y, sin2_f<INLINE_SLOW>(y1), x.y);
        o.z = fmaf(ia.z, sin2_f<INLINE_SLOW>(y2), x.z); o.w = fmaf(ia.w, sin2_f<INLINE_SLOW>(y3), x.w);
    } else {
        o.x = fmaf(ia.x, sin2_poly(y0), x.x); o.y = fmaf(ia.y, sin2_poly(y1), x.y);
        o.z = fmaf(ia.z, sin2_poly(y2), x.z); o.w = fmaf(ia.w, sin2_poly(y3), x.w);
    }
    return o;
}
// Decoder-class Snake (layers downstream of the VQ whose operands are rounded to 16 mantissa bits anyway): same
// reduction mod pi, then the SFU sine (MUFU.SIN, abs error ~4e-7 on [-pi/2, pi/2]) instead of the polynomial.
// 9 instructions per element instead of 15; never used upstream of the VQ.
__device__ __forceinline__ float sin2_mufu(float x) {
    float k = rintf(x * 0.318309886183790672f);
    float r = fmaf(k, -3.14159274101257324f, x);
    r = fmaf(k, 8.74227765734758578e-8f, r);
    float s = __sinf(r);
    return s * s;
}
__device__ __forceinline__ float4 snake4_mufu(float4 x, float4 al, float4 ia) {
    float4 o;
    o.x = fmaf(ia.x, sin2_mufu(al.x * x.x), x.x); o.y = fmaf(ia.y, sin2_mufu(al.y * x.y), x.y);
    o.z = fmaf(ia.z, sin2_mufu(al.z * x.z), x.z); o.w = fmaf(ia.w, sin2_mufu(al.w * x.w), x.w);
    return o;
}
template <bool MUFU, bool INLINE_SLOW = false>
__device__ __forceinline__ float4 snake4_sel(float4 x, float4 al, float4 ia) {
    if constexpr (MUFU) return snake4_mufu(x, al, ia);
    else return snake4<INLINE_SLOW>(x, al, ia);
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// x * tanh(softplus(x)), modules/style_encoder.py:6-10 ; F.softplus threshold 20
__device__ __forceinline__ float mish_f(float x) {
    float sp = x > 20.0f ? x : log1pf(expf(x));
    return x * tanhf(sp);
}

enum OutAct { ACT_NONE = 0, ACT_TANH = 1, ACT_MISH = 2, ACT_SNAKE = 3, ACT_LRELU = 4 };

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace fac
