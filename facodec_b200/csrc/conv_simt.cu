// Generic channels-last 1-D convolution as an implicit GEMM on the fp32 FMA pipe.
//
// Replaces the reference's F.pad(reflect) + nn.Conv1d / nn.ConvTranspose1d / nn.Linear call
// sites (dac/model/encodec.py:212-228 SConv1d.forward, :248-270 SConvTranspose1d.forward,
// modules/style_encoder.py, modules/wavenet.py:145-160, nn.LSTM input projections) with one
// kernel:
//
//   y[b][t][co] = epi( bias[co] + sum_{tap<K} sum_{ci<Cin}
//                      pro(x[b][map(t*stride + tap*dil - pad_left)][ci]) * w[tap*Cin + ci][co] )
//
// * x, y channels-last fp32; w packed "kk-major" [K*Cin][ldw] (ldw = Cout rounded up to 4).
// * map() = reflect / zero padding index map (common.cuh PadMap) -- no padded copy in HBM.
// * pro() = optional Snake on the input (dac/nn/layers.py:17-24), per input channel.
// * epi() = bias, then optional Snake / tanh / Mish, then optional residual add, optional
//   row mask (t < valid_len[b]), optional transposed ([B][Cout][T]) store.
// * ConvTranspose1d(k=2s, stride=s) + right trim is run as a K=2 zero-left-padded conv with
//   Cout*s output channels (phase-major); [B][T][s*Cout] IS [B][T*s][Cout] in channels-last.
//
// Tile: 128 (time) x BN (channels) per CTA, 8x8 register tile per thread, BK=16 deep smem
// stages with register prefetch of the next stage.  This is the fp32-exact path (bit-exact VQ
// indices need fp32-faithful accumulation, SURVEY.md section 0.5).
#include "common.cuh"
#include "kernels.h"

namespace fac {

constexpr int CONV_BM = 128;
constexpr int CONV_BK = 16;
constexpr int CONV_XPAD = 4;

template <int BN>
__global__ void __launch_bounds__(2 * BN) conv_cl_kernel(ConvParams p) {
    constexpr int BM = CONV_BM, BK = CONV_BK;
    constexpr int NT = 2 * BN;               // 16 t-groups x BN/8 co-groups
    constexpr int CG = BN / 8;               // co groups
    constexpr int LC = (CG % 8 == 0) ? 8 : 4; // lanes along co inside a warp
    constexpr int LT = 32 / LC;              // lanes along t
    constexpr int WC = CG / LC;              // warps along co
    constexpr int A_F4 = BM * BK / 4;        // float4 per A stage
    constexpr int A_PER = (A_F4 + NT - 1) / NT;
    constexpr int W_F4 = BK * BN / 4;
    constexpr int W_PER = W_F4 / NT;         // == 2

    __shared__ __align__(16) float xs[BK][BM + CONV_XPAD];
    __shared__ __align__(16) float ws[BK][BN];

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int wc = warp % WC, wt = warp / WC;
    const int cg = wc * LC + (lane % LC);    // co group 0..CG-1
    const int tg = wt * LT + (lane / LC);    // t group 0..15
    const int b = blockIdx.z;
    const int t0 = blockIdx.x * BM;
    const int co0 = blockIdx.y * BN;

    const float* __restrict__ xb = p.x + (size_t)b * p.x_bstride;
    const PadMap pm = PadMap::lane(p.lane_len, b, p.Tin, p.pad_left, p.pad_right, p.pad_reflect);
    const int Ktot = p.K * p.Cin;
    const bool vec_a = (p.Cin % 4) == 0;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    float4 a_reg[A_PER];
    float4 w_reg[W_PER];

    auto load_stage = [&](int kk0) {
#pragma unroll
        for (int it = 0; it < A_PER; ++it) {
            int i = tid + it * NT;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < A_F4) {
                int r = i >> 2, c4 = i & 3;
                int kk = kk0 + c4 * 4;
                int t = t0 + r;
                if (t < p.Tout && kk < Ktot) {
                    if (vec_a) {
                        int tap = kk / p.Cin, ci = kk - tap * p.Cin;
                        int row = pm.src(t * p.stride + tap * p.dil - p.pad_left);
                        if (row >= 0) {
                            v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)row * p.ldx + ci));
                            if (p.in_alpha) {
                                float4 al = __ldg(reinterpret_cast<const float4*>(p.in_alpha + ci));
                                float4 ia = __ldg(reinterpret_cast<const float4*>(p.in_inv_alpha + ci));
                                v.x = snake_f(v.x, al.x, ia.x);
                                v.y = snake_f(v.y, al.y, ia.y);
                                v.z = snake_f(v.z, al.z, ia.z);
                                v.w = snake_f(v.w, al.w, ia.w);
                            }
                        }
                    } else {
                        float e[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            int k2 = kk + j;
                            float val = 0.f;
                            if (k2 < Ktot) {
                                int tap = k2 / p.Cin, ci = k2 - tap * p.Cin;
                                int row = pm.src(t * p.stride + tap * p.dil - p.pad_left);
                                if (row >= 0) {
                                    val = __ldg(xb + (size_t)row * p.ldx + ci);
                                    if (p.in_alpha) val = snake_f(val, p.in_alpha[ci], p.in_inv_alpha[ci]);
                                }
                            }
                            e[j] = val;
                        }
                        v = make_float4(e[0], e[1], e[2], e[3]);
                    }
                }
            }
            a_reg[it] = v;
        }
#pragma unroll
        for (int it = 0; it < W_PER; ++it) {
            int i = tid + it * NT;
            int kr = i / (BN / 4), c4 = i % (BN / 4);
            int kk = kk0 + kr;
            int co = co0 + c4 * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kk < Ktot && co < p.ldw) v = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)kk * p.ldw + co));
            w_reg[it] = v;
        }
    };
    auto store_stage = [&]() {
#pragma unroll
        for (int it = 0; it < A_PER; ++it) {
            int i = tid + it * NT;
            if (i < A_F4) {
                int r = i >> 2, c4 = i & 3;
                xs[c4 * 4 + 0][r] = a_reg[it].x;
                xs[c4 * 4 + 1][r] = a_reg[it].y;
                xs[c4 * 4 + 2][r] = a_reg[it].z;
                xs[c4 * 4 + 3][r] = a_reg[it].w;
            }
        }
#pragma unroll
        for (int it = 0; it < W_PER; ++it) {
            int i = tid + it * NT;
            int kr = i / (BN / 4), c4 = i % (BN / 4);
            *reinterpret_cast<float4*>(&ws[kr][c4 * 4]) = w_reg[it];
        }
    };

    const int nstage = (Ktot + BK - 1) / BK;
    load_stage(0);
    for (int s = 0; s < nstage; ++s) {
        __syncthreads();   // previous stage fully consumed
        store_stage();
        __syncthreads();
        if (s + 1 < nstage) load_stage((s + 1) * BK);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float4 a0 = *reinterpret_cast<const float4*>(&xs[kk][tg * 8]);
            float4 a1 = *reinterpret_cast<const float4*>(&xs[kk][tg * 8 + 4]);
            float4 b0 = *reinterpret_cast<const float4*>(&ws[kk][cg * 8]);
            float4 b1 = *reinterpret_cast<const float4*>(&ws[kk][cg * 8 + 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
    }

    // ---- epilogue ----
    const int cbase = co0 + cg * 8;
    if (cbase >= p.Cout) return;
    float bias[8], oal[8], oia[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int co = cbase + j;
        bool ok = co < p.Cout;
        bias[j] = (p.bias && ok) ? p.bias[co] : 0.f;
        oal[j] = (p.out_act == ACT_SNAKE && ok) ? p.out_alpha[co] : 0.f;
        oia[j] = (p.out_act == ACT_SNAKE && ok) ? p.out_inv_alpha[co] : 0.f;
    }
    const int vlen = p.valid_len ? p.valid_len[b] : 0x7fffffff;
    float* __restrict__ yb = p.y + (size_t)b * p.y_bstride;
    const float* __restrict__ rb = p.res ? p.res + (size_t)b * p.y_bstride : nullptr;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int t = t0 + tg * 8 + i;
        if (t >= p.Tout) break;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float o = acc[i][j] + bias[j];
            if (p.out_act == ACT_TANH) o = tanhf(o);
            else if (p.out_act == ACT_MISH) o = mish_f(o);
            else if (p.out_act == ACT_SNAKE) o = snake_f(o, oal[j], oia[j]);
            v[j] = o;
        }
        if (p.y_transposed) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (cbase + j < p.Cout) yb[(size_t)(cbase + j) * p.Tout + t] = (t < vlen) ? v[j] : 0.f;
            continue;
        }
        size_t off = (size_t)t * p.ldy + cbase;
        if (rb) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (cbase + j < p.Cout) v[j] += rb[off + j];
        }
        if (t >= vlen) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = 0.f;
        }
        if (cbase + 8 <= p.Cout && (p.ldy % 4) == 0) {
            *reinterpret_cast<float4*>(yb + off) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(yb + off + 4) = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (cbase + j < p.Cout) yb[off + j] = v[j];
        }
    }
}

// ---- Cout == 1 (decoder's last conv, dac.py:158-160: Snake -> SConv1d(96 -> 1, k=7) -> tanh) -------
// A dot product of K*Cin per output sample: HBM-bound (reads the widest activation of the model once).
// CTA = 128 output samples: stage the (128 + halo) x Cin input tile in shared memory with Snake applied
// (coalesced 16-byte loads, 4 in flight per thread).  Then thread (t, h) accumulates output sample t over
// the 16-byte channel pieces c4 = h, h+2, ... of every tap with 128-bit shared loads: the row pitch Cp is
// 4*odd floats, so the 8 threads of a quarter-warp (consecutive t, same piece) hit 8 distinct bank groups;
// weights are warp-uniform broadcasts.  The two halves meet in shared memory; stores are coalesced.
constexpr int C1_TILE = 128;
__host__ __device__ inline int c1_pitch(int Cin) { return ((Cin / 4) & 1) ? Cin : Cin + 4; }
__global__ void __launch_bounds__(256) conv_cout1_kernel(ConvParams p) {
    extern __shared__ __align__(16) float c1_smem[];
    const int Cin = p.Cin, Cp = c1_pitch(Cin);
    const int halo = (p.K - 1) * p.dil;
    const int rows = C1_TILE + halo;
    float* xs = c1_smem;                        // [rows][Cp]
    float* wsm = c1_smem + (size_t)rows * Cp;   // [K][Cin]
    float* part = wsm + (size_t)p.K * Cin;      // [C1_TILE] partial sums of the odd pieces
    const int b = blockIdx.y, t0 = blockIdx.x * C1_TILE;
    const float* __restrict__ xb = p.x + (size_t)b * p.x_bstride;
    const PadMap pm = PadMap::lane(p.lane_len, b, p.Tin, p.pad_left, p.pad_right, p.pad_reflect);
    const int c4n = Cin / 4;
    const bool has_alpha = p.in_alpha != nullptr;
    const int total = rows * c4n;
    for (int i0 = threadIdx.x; i0 < total; i0 += 4 * 256) {
        float4 v[4];
        int rr[4], cc[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u * 256;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            rr[u] = -1; cc[u] = 0;
            if (i < total) {
                const int r = i / c4n, c4 = i - r * c4n;
                rr[u] = r; cc[u] = c4;
                const int row = pm.src(t0 + r - p.pad_left);
                if (row >= 0 && t0 + r - halo < p.Tout) v[u] = __ldg(reinterpret_cast<const float4*>(xb + (size_t)row * p.ldx + c4 * 4));
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (rr[u] < 0) continue;
            float4 x4 = v[u];
            if (has_alpha) {
                const float4 al = __ldg(reinterpret_cast<const float4*>(p.in_alpha + cc[u] * 4));
                const float4 ia = __ldg(reinterpret_cast<const float4*>(p.in_inv_alpha + cc[u] * 4));
                x4.x = snake_fast(x4.x, al.x, ia.x); x4.y = snake_fast(x4.y, al.y, ia.y);
                x4.z = snake_fast(x4.z, al.z, ia.z); x4.w = snake_fast(x4.w, al.w, ia.w);
            }
            *reinterpret_cast<float4*>(xs + (size_t)rr[u] * Cp + cc[u] * 4) = x4;
        }
    }
    for (int i = threadIdx.x; i < p.K * Cin; i += 256) wsm[i] = p.w[(size_t)i * p.ldw];
    __syncthreads();
    const int tl = threadIdx.x & (C1_TILE - 1), h = threadIdx.x >> 7;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int tap = 0; tap < p.K; ++tap) {
        const float* xr = xs + (size_t)(tl + tap * p.dil) * Cp;
        const float* wr = wsm + tap * Cin;
#pragma unroll 4
        for (int c4 = h; c4 < c4n; c4 += 2) {
            const float4 xv = *reinterpret_cast<const float4*>(xr + c4 * 4);
            const float4 wv = *reinterpret_cast<const float4*>(wr + c4 * 4);
            a0 = fmaf(xv.x, wv.x, a0); a1 = fmaf(xv.y, wv.y, a1);
            a2 = fmaf(xv.z, wv.z, a2); a3 = fmaf(xv.w, wv.w, a3);
        }
    }
    const float acc = (a0 + a1) + (a2 + a3);
    if (h == 1) part[tl] = acc;
    __syncthreads();
    if (h == 0) {
        const int t = t0 + tl;
        if (t < p.Tout) {
            float v = acc + part[tl] + (p.bias ? p.bias[0] : 0.f);
            if (p.out_act == ACT_TANH) v = tanhf(v);
            p.y[(size_t)b * p.y_bstride + (size_t)t * p.ldy] = v;
        }
    }
}

// ---- Cin == 1 (encoder's first conv, dac.py:79: SConv1d(1 -> 64, k=7)) ------------------------------
// K FMAs per output and a 4*Cout-byte row to write per input sample: purely HBM-write-bound (786 MB at B=32).
// CTA = C1I_T consecutive samples; thread (r, c4) keeps the K weights of its 4 channels in registers and walks the
// tile's rows r, r + 256/(Cout/4), ...: the Cout/4 threads of a row write it as one contiguous segment.
constexpr int C1I_T = 256;
constexpr int C1I_MAXK = 16;
__global__ void __launch_bounds__(256) conv_cin1_kernel(ConvParams p) {
    __shared__ float xs[C1I_T + C1I_MAXK * 16];
    const int halo = (p.K - 1) * p.dil;
    const int b = blockIdx.y, t0 = blockIdx.x * C1I_T;
    const float* __restrict__ xb = p.x + (size_t)b * p.x_bstride;
    const PadMap pm = PadMap::lane(p.lane_len, b, p.Tin, p.pad_left, p.pad_right, p.pad_reflect);
    for (int i = threadIdx.x; i < C1I_T + halo; i += 256) {
        const int src = pm.src(t0 + i - p.pad_left);
        float v = src >= 0 ? __ldg(xb + (size_t)src * p.ldx) : 0.f;
        if (p.in_alpha) v = snake_fast(v, p.in_alpha[0], p.in_inv_alpha[0]);
        xs[i] = v;
    }
    const int c4n = p.Cout / 4, rows_per_pass = 256 / c4n;
    const int c4 = threadIdx.x % c4n, r0 = threadIdx.x / c4n;
    float4 w[C1I_MAXK];
#pragma unroll
    for (int k = 0; k < C1I_MAXK; ++k)
        w[k] = k < p.K ? __ldg(reinterpret_cast<const float4*>(p.w + (size_t)k * p.ldw + c4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 bi = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + c4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    if (r0 >= rows_per_pass) return;
    float* __restrict__ yb = p.y + (size_t)b * p.y_bstride;
    for (int r = r0; r < C1I_T; r += rows_per_pass) {
        const int t = t0 + r;
        if (t >= p.Tout) break;
        float4 a = bi;
#pragma unroll
        for (int k = 0; k < C1I_MAXK; ++k)
            if (k < p.K) {
                const float xv = xs[r + k * p.dil];
                a.x = fmaf(xv, w[k].x, a.x); a.y = fmaf(xv, w[k].y, a.y);
                a.z = fmaf(xv, w[k].z, a.z); a.w = fmaf(xv, w[k].w, a.w);
            }
        if (p.out_act == ACT_TANH) { a.x = tanhf(a.x); a.y = tanhf(a.y); a.z = tanhf(a.z); a.w = tanhf(a.w); }
        *reinterpret_cast<float4*>(yb + (size_t)t * p.ldy + c4 * 4) = a;
    }
}

cudaError_t launch_conv(const ConvParams& p, cudaStream_t st) {
    if (p.Tout <= 0 || p.B <= 0) return cudaSuccess;
    if (p.Cin == 1 && p.stride == 1 && p.K <= C1I_MAXK && (p.K - 1) * p.dil <= C1I_MAXK * 16 && (p.Cout % 4) == 0 &&
        p.Cout <= 1024 && (256 % (p.Cout / 4)) == 0 && (p.ldw % 4) == 0 && (p.ldy % 4) == 0 && !p.res && !p.valid_len &&
        !p.y_transposed && (p.out_act == ACT_NONE || p.out_act == ACT_TANH)) {
        dim3 grid((p.Tout + C1I_T - 1) / C1I_T, p.B);
        conv_cin1_kernel<<<grid, 256, 0, st>>>(p);
        return cudaGetLastError();
    }
    if (p.Cout == 1 && p.stride == 1 && (p.Cin % 4) == 0 && !p.res && !p.valid_len && !p.y_transposed &&
        (p.out_act == ACT_NONE || p.out_act == ACT_TANH)) {
        size_t smem = sizeof(float) * ((size_t)(C1_TILE + (p.K - 1) * p.dil) * c1_pitch(p.Cin) + (size_t)p.K * p.Cin + C1_TILE);
        if (smem <= 200 * 1024) {
            // function attributes are per device (a process may hold handles on several GPUs): set it on every launch of this
            // once-per-forward kernel instead of caching a process-wide flag
            cudaError_t e = cudaFuncSetAttribute(conv_cout1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
            if (e != cudaSuccess) return e;
            dim3 grid((p.Tout + C1_TILE - 1) / C1_TILE, p.B);
            conv_cout1_kernel<<<grid, 256, smem, st>>>(p);
            return cudaGetLastError();
        }
    }
    dim3 grid((p.Tout + CONV_BM - 1) / CONV_BM, 1, p.B);
    // channel tile with the least padding waste (ties -> wider tile)
    auto padded = [&](int bn) { return (p.Cout + bn - 1) / bn * bn; };
    int bn = 128;
    if (padded(96) < padded(bn)) bn = 96;
    if (padded(64) < padded(bn)) bn = 64;
    grid.y = (p.Cout + bn - 1) / bn;
    if (bn == 128) conv_cl_kernel<128><<<grid, 256, 0, st>>>(p);
    else if (bn == 96) conv_cl_kernel<96><<<grid, 192, 0, st>>>(p);
    else conv_cl_kernel<64><<<grid, 128, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace fac
