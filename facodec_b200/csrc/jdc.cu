// JDCNet (modules/JDC/model.py, eval mode) small kernels around the 3x3 convs of conv2d_tc_kernel, and train.py's F0 and
// energy targets (train.py:214-254).
//
// Feature maps are channels-last [B][T][F + 2][C]: frequency columns 0 and F + 1 are zero, so that a 3x3 conv over the map
// flattened to rows of C channels is a 9-tap row-offset conv (conv_tc.cu, row2d = F + 2).  Every kernel here writes those
// columns as zeros.  Lane b of a batch is its own first len[b] frames; a frame t >= len[b] of an intermediate map is a
// finite don't-care (no conv reads it: the convs zero-pad time at each lane's own end), and of an output is zero.
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace fac {

namespace {

__device__ __forceinline__ float lrelu(float v) { return v >= 0.f ? v : 0.01f * v; }

// conv_block[0..2]: Conv2d(1, 64, 3, padding=1) with its BatchNorm folded into w / bias, then LeakyReLU.
// mel [B][80][T] -> y [B][T][82][64].  One thread per (frame, column, 4 channels), the channel quad fastest: a warp's
// stores are 512 contiguous bytes, and its 9 mel loads touch two columns.
__global__ void jdc_conv_in_kernel(const float* __restrict__ mel, const float* __restrict__ w /*[9][64]*/,
                                   const float* __restrict__ bias, float* __restrict__ y, int B, int T, const int* lens) {
    __shared__ float ws[9 * 64 + 64];
    for (int i = threadIdx.x; i < 9 * 64; i += blockDim.x) ws[i] = w[i];
    for (int i = threadIdx.x; i < 64; i += blockDim.x) ws[9 * 64 + i] = bias[i];
    __syncthreads();
    const int b = blockIdx.y;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)T * 82 * 16) return;
    const int q = (int)(idx & 15);
    const long long r = idx >> 4;
    const int t = (int)(r / 82), j = (int)(r % 82);
    const int L = lens ? lens[b] : T;
    float4* yo = reinterpret_cast<float4*>(y + (((size_t)b * T + t) * 82 + j) * 64) + q;
    if (j == 0 || j == 81) {
        *yo = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const int f = j - 1;
    float xin[9];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
            const int tt = t + kh - 1, ff = f + kw - 1;
            xin[kh * 3 + kw] = (tt >= 0 && tt < L && ff >= 0 && ff < 80) ? __ldg(mel + ((size_t)b * 80 + ff) * T + tt) : 0.f;
        }
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int co = 4 * q + e;
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) s = fmaf(xin[k], ws[k * 64 + co], s);
        o[e] = lrelu(s + ws[9 * 64 + co]);
    }
    *yo = make_float4(o[0], o[1], o[2], o[3]);
}

// ResBlock.pre_conv: BatchNorm2d (eval, as scale / shift) + LeakyReLU + MaxPool2d((1, 2)).
// x [B][T][F + 2][C] -> y [B][T][F/2 + 2][C]
__global__ void jdc_pre_pool_kernel(const float* __restrict__ x, const float* __restrict__ sc, const float* __restrict__ sh,
                                    float* __restrict__ y, int B, int T, int F, int C) {
    const int Fo = F / 2, C4 = C / 4;
    const long long n = (long long)B * T * (Fo + 2) * C4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const long long r = i / C4;
        const int j = (int)(r % (Fo + 2));
        const long long bt = r / (Fo + 2);
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j > 0 && j <= Fo) {
            const int f0 = 2 * (j - 1);
            const float4 s = __ldg(reinterpret_cast<const float4*>(sc) + c4), h = __ldg(reinterpret_cast<const float4*>(sh) + c4);
            const float4* xr = reinterpret_cast<const float4*>(x + (bt * (F + 2) + f0 + 1) * C) + c4;
            const float4 a = xr[0], b2 = xr[C4];
            o.x = fmaxf(lrelu(fmaf(a.x, s.x, h.x)), lrelu(fmaf(b2.x, s.x, h.x)));
            o.y = fmaxf(lrelu(fmaf(a.y, s.y, h.y)), lrelu(fmaf(b2.y, s.y, h.y)));
            o.z = fmaxf(lrelu(fmaf(a.z, s.z, h.z)), lrelu(fmaf(b2.z, s.z, h.z)));
            o.w = fmaxf(lrelu(fmaf(a.w, s.w, h.w)), lrelu(fmaf(b2.w, s.w, h.w)));
        }
        reinterpret_cast<float4*>(y + (r * C))[c4] = o;
    }
}

// pool_block in eval mode: BatchNorm2d + LeakyReLU (-> GAN_feature [B][256][10][T]), MaxPool2d((1, 4)) (-> pool_out
// [B][256][T][2]; Dropout is the identity), and the BiLSTM input [B][T][512] at c * 2 + k (model.py:127's permute / view).
// x [B][T][12][256].  One block per 32 frames x 32 channels: the tile goes through shared memory, so that the loads run
// along channels and each output's stores along its own contiguous axis.
constexpr int kPoolTile = 32;
__global__ void jdc_pool_block_kernel(const float* __restrict__ x, const float* __restrict__ sc, const float* __restrict__ sh,
                                      float* __restrict__ gan, float* __restrict__ pool, float* __restrict__ lstm_in, int B, int T,
                                      const int* lens) {
    __shared__ float v[10][kPoolTile][kPoolTile + 1];      // [f][frame][channel]
    const int t0 = blockIdx.x * kPoolTile, c0 = blockIdx.y * kPoolTile, b = blockIdx.z;
    const int L = lens ? lens[b] : T;
    for (int i = threadIdx.x; i < kPoolTile * 10 * kPoolTile; i += blockDim.x) {
        const int c = i % kPoolTile, f = (i / kPoolTile) % 10, tl = i / (kPoolTile * 10), t = t0 + tl;
        float o = 0.f;
        if (t < L) o = lrelu(fmaf(x[(((size_t)b * T + t) * 12 + f + 1) * 256 + c0 + c], __ldg(sc + c0 + c), __ldg(sh + c0 + c)));
        v[f][tl][c] = o;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kPoolTile * 10 * kPoolTile; i += blockDim.x) {
        const int tl = i % kPoolTile, f = (i / kPoolTile) % 10, c = i / (kPoolTile * 10), t = t0 + tl;
        if (t < T) gan[(((size_t)b * 256 + c0 + c) * 10 + f) * T + t] = v[f][tl][c];
    }
    auto mx = [&](int tl, int c, int k) {
        return fmaxf(fmaxf(v[4 * k][tl][c], v[4 * k + 1][tl][c]), fmaxf(v[4 * k + 2][tl][c], v[4 * k + 3][tl][c]));
    };
    for (int i = threadIdx.x; i < kPoolTile * kPoolTile; i += blockDim.x) {
        const int tl = i % kPoolTile, c = i / kPoolTile, t = t0 + tl;
        if (t < T) *reinterpret_cast<float2*>(pool + (((size_t)b * 256 + c0 + c) * T + t) * 2) = make_float2(mx(tl, c, 0), mx(tl, c, 1));
    }
    for (int i = threadIdx.x; i < kPoolTile * kPoolTile; i += blockDim.x) {
        const int c = i % kPoolTile, tl = i / kPoolTile, t = t0 + tl;
        if (t < T) *reinterpret_cast<float2*>(lstm_in + ((size_t)b * T + t) * 512 + 2 * (c0 + c)) = make_float2(mx(tl, c, 0), mx(tl, c, 1));
    }
}

// classifier (Linear(512, 1)) + abs over [forward h | reverse h]: one warp per frame, a fixed-order sum (lane partials of
// 16 consecutive features, then a butterfly), so the result does not depend on B.
__global__ void jdc_head_kernel(const float* __restrict__ yf, const float* __restrict__ yb, const float* __restrict__ w,
                                const float* __restrict__ bias, float* __restrict__ f0, int B, int T, const int* lens) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * T) return;
    const int b = warp / T, t = warp % T;
    const float* src = (lane < 16 ? yf : yb) + (size_t)warp * 256 + (lane & 15) * 16;
    const float* wl = w + lane * 16;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) s = fmaf(src[k], __ldg(wl + k), s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) f0[warp] = t < (lens ? lens[b] : T) ? fabsf(s + __ldg(bias)) : 0.f;
}

// block-wide sum of one value per thread in a fixed tree order (256 threads)
__device__ float block_sum(float v, float* red) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const float r = red[0];
    __syncthreads();
    return r;
}

// train.py:223-251 per lane: voiced = F0 > 5, log2, (x - mean) / std (unbiased), -10 on unvoiced frames, NaN / inf -> -10;
// glob = mean, 0 without a voiced frame.  One 256-thread block per lane; frames t >= len[b] are -10 and count for nothing.
__global__ void f0_targets_kernel(const float* __restrict__ f0, const int* lens, int T, float* __restrict__ out,
                                  float* __restrict__ glob) {
    __shared__ float red[256];
    const int b = blockIdx.x;
    const int L = lens ? lens[b] : T;
    const float* x = f0 + (size_t)b * T;
    float n = 0.f, s = 0.f;
    for (int t = threadIdx.x; t < L; t += 256)
        if (x[t] > 5.0f) { n += 1.f; s += log2f(x[t]); }
    n = block_sum(n, red);
    s = block_sum(s, red);
    const float mean = s / n;
    float q = 0.f;
    for (int t = threadIdx.x; t < L; t += 256)
        if (x[t] > 5.0f) { const float d = log2f(x[t]) - mean; q = fmaf(d, d, q); }
    q = block_sum(q, red);
    const float sd = sqrtf(q / (n - 1.f));      // n = 1: 0 / 0 = NaN, as torch.std gives
    for (int t = threadIdx.x; t < T; t += 256) {
        float v = -10.f;
        if (t < L && x[t] > 5.0f) v = (log2f(x[t]) - mean) / sd;
        if (isnan(v) || isinf(v)) v = -10.f;
        out[(size_t)b * T + t] = v;
    }
    if (threadIdx.x == 0) glob[b] = n > 0.f ? mean : 0.f;
}

// modules/commons.py:176-181 log_norm(x, mean=-4, std=4, dim=2) on mel [B][80][T]: log(||exp(x * 4 - 4)||_2 over the bins)
__global__ void log_norm_kernel(const float* __restrict__ mel, int B, int T, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * T) return;
    const int b = (int)(i / T), t = (int)(i % T);
    float s = 0.f;
    for (int k = 0; k < 80; ++k) {
        const float e = expf(__fadd_rn(__fmul_rn(mel[((size_t)b * 80 + k) * T + t], 4.f), -4.f));
        s = fmaf(e, e, s);
    }
    out[i] = logf(sqrtf(s));
}

}  // namespace

cudaError_t launch_jdc_conv_in(const float* mel, const float* w, const float* bias, float* y, int B, int T, const int* lens,
                               cudaStream_t st) {
    if (B <= 0 || T <= 0) return cudaSuccess;
    dim3 grid((unsigned)(((long long)T * 82 * 16 + 255) / 256), B);
    jdc_conv_in_kernel<<<grid, 256, 0, st>>>(mel, w, bias, y, B, T, lens);
    return cudaGetLastError();
}

cudaError_t launch_jdc_pre_pool(const float* x, const float* sc, const float* sh, float* y, int B, int T, int F, int C,
                                cudaStream_t st) {
    if (C % 4 || F % 2) return cudaErrorInvalidValue;
    const long long n = (long long)B * T * (F / 2 + 2) * (C / 4);
    if (n <= 0) return cudaSuccess;
    const long long blocks = (n + 255) / 256;
    jdc_pre_pool_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 256, 0, st>>>(x, sc, sh, y, B, T, F, C);
    return cudaGetLastError();
}

cudaError_t launch_jdc_pool_block(const float* x, const float* sc, const float* sh, float* gan, float* pool, float* lstm_in,
                                  int B, int T, const int* lens, cudaStream_t st) {
    if (B <= 0 || T <= 0) return cudaSuccess;
    jdc_pool_block_kernel<<<dim3((T + kPoolTile - 1) / kPoolTile, 256 / kPoolTile, B), 256, 0, st>>>(x, sc, sh, gan, pool, lstm_in,
                                                                                                   B, T, lens);
    return cudaGetLastError();
}

cudaError_t launch_jdc_head(const float* yf, const float* yb, const float* w, const float* bias, float* f0, int B, int T,
                            const int* lens, cudaStream_t st) {
    const long long n = (long long)B * T * 32;
    if (n <= 0) return cudaSuccess;
    jdc_head_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(yf, yb, w, bias, f0, B, T, lens);
    return cudaGetLastError();
}

cudaError_t launch_f0_targets(const float* f0, const int* lens, int B, int T, float* out, float* glob, cudaStream_t st) {
    if (B <= 0 || T <= 0) return cudaSuccess;
    f0_targets_kernel<<<B, 256, 0, st>>>(f0, lens, T, out, glob);
    return cudaGetLastError();
}

cudaError_t launch_log_norm(const float* mel, int B, int T, float* out, cudaStream_t st) {
    const long long n = (long long)B * T;
    if (n <= 0) return cudaSuccess;
    log_norm_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(mel, B, T, out);
    return cudaGetLastError();
}

}  // namespace fac
