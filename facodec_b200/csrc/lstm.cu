// Persistent LSTM recurrence for SLSTM (dac/model/encodec.py:272-288 -> nn.LSTM(C, C, 2)).
//
// The input projections x W_ih^T + b_ih + b_hh for all T steps are one GEMM (conv_simt.cu);
// what remains is the serial chain  gates_t = xg_t + h_{t-1} W_hh^T  for T steps.  One
// cooperative launch runs all T steps of one layer: G = H/U CTAs, CTA c owns hidden units
// [c*U, c*U+U) (all four gates), keeps their cell state in shared memory, and exchanges h_t
// through a [2][H][32] buffer in L2 with one device-wide barrier per step.
//
// Per step each CTA computes a [4U gate rows] x [32 batch] x [H] product: the 8 warps split H
// eight ways and stream their slice of W_hh (pre-packed per CTA as [H][4U], so the copy is
// linear) and of h_{t-1} through private multi-stage cp.async rings, and feed them to the tensor
// cores as mma.sync m16n8k8 TF32 tiles with the same fp32-faithful 3xTF32 split as the convs
// (hi/lo formed in registers; 48-72 chained MMAs per accumulator, then an fp32 cross-warp sum).
// A 32 x 4U x H product per step is far too small for a wgmma tile pipeline.  Measured per
// step (clock64 probe, fac_debug_lstm_phase_clocks): barrier wait ~2.0k cycles, K loop 12k (H=1024) /
// 23.5k (H=1536), reduce+gates 1.4-2.6k, publish 1.4k.  The K loop is bound by the legacy HMMA.1688
// TF32 rate of this chip (~1 per 32 cycles per SM sub-partition == the fp32 FMA rate: the earlier FMA
// version of this loop ran at the same speed), not by the cp.async ring (deepening it changed nothing).  Partial sums meet in
// shared memory, then 32*U threads apply the gate math (PyTorch gate order i, f, g, o).
#include <cooperative_groups.h>
#include "common.cuh"
#include "kernels.h"

namespace fac {

// accumulated clock64 per phase of CTA 0 (kernel-tuning aid): [0] barrier wait, [1] K loop, [2] reduce+gates, [3] publish
__device__ long long g_lstm_phase_clock[4];

constexpr int LSTM_BT = 32;     // batch tile (columns of hT)
constexpr int LSTM_WARPS = 8;
constexpr int LSTM_KS = 16;     // k rows per cp.async sub-chunk
// cp.async pipeline depth (stages per warp): as deep as shared memory allows -- the K loop is bound by
// bytes in flight x L2 latency, not by the MMAs.  The cross-warp reduction buffer aliases the stage memory.
template <int U> struct LstmDepth { static constexpr int D = (U == 8) ? 5 : 4; };
// padded smem row of the h sub-chunk (conflict-free B fragments): TF32 fragments read rows k0+t and k0+t+4
// (pitch 40: 8t + g), bf16 fragments read row pairs 2t, 2t+1 (pitch 36: 2*36*t = 8t mod 32)
template <bool BF16> struct LstmHP { static constexpr int V = BF16 ? LSTM_BT + 4 : LSTM_BT + 8; };

__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const float (&a)[4], const float (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
          "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}

__device__ __forceinline__ void mma_bf16_16x8x16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// (x0, x1) -> bf16x2 hi word (x0 in the low half) and the bf16x2 word of the residuals
__device__ __forceinline__ void bf16_split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    const float h0 = __uint_as_float(hi << 16), h1 = __uint_as_float(hi & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - h1), "f"(x0 - h0));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// BF16 = true (layers downstream of the VQ only): W_hh arrives pre-split into bf16 hi / bf16 lo words (two
// consecutive k per 32-bit word, per 16-k sub-chunk [hi|lo][8 k-pairs][4U]), h is split in registers, and the
// product runs as 3 m16n8k16 bf16 MMAs per 16 k instead of 6 m16n8k8 TF32 MMAs (the K loop is HMMA-bound).
template <int U, bool BF16>
__global__ void __launch_bounds__(LSTM_WARPS * 32, 1) lstm_rec_kernel(LstmParams p) {
    constexpr int LSTM_HP = LstmHP<BF16>::V;
    constexpr int R = 4 * U;
    constexpr int RP = R + 1;   // padded row of the reduction buffer (bank-conflict-free reads)
    constexpr int WP = R + 8;                   // padded smem row of the W sub-chunk
    constexpr int MT = R / 16, NTL = LSTM_BT / 8;
    constexpr int STAGE_F = LSTM_KS * (LSTM_HP + WP);  // floats per stage per warp
    constexpr int LSTM_D = LstmDepth<U>::D;
    static_assert(LSTM_D * STAGE_F >= LSTM_BT * RP, "reduction buffer must fit in a warp's own stage memory");
    extern __shared__ __align__(16) float smem[];
    float* stage_base = smem;                                   // [8 warps][LSTM_D][STAGE_F]
    float* cstate = smem + LSTM_WARPS * LSTM_D * STAGE_F;       // [32][U]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x;
    const int j0 = cta * U;
    const int H = p.H;
    const int kslice = H / LSTM_WARPS;
    const int k_begin = warp * kslice;
    const int nsub = kslice / LSTM_KS;
    const int fg = lane >> 2, ft = lane & 3;   // mma fragment coordinates

    for (int i = tid; i < LSTM_BT * U; i += blockDim.x) cstate[i] = 0.f;
    __syncthreads();

    const float* wsrc = (BF16 ? p.whh_p16 : p.whh_p) + (size_t)cta * H * R;
    float* my_stage = stage_base + warp * LSTM_D * STAGE_F;

    constexpr int PAIRS = (LSTM_BT * U + LSTM_WARPS * 32 - 1) / (LSTM_WARPS * 32);
    const bool probe = (cta == 0 && tid == 0);
    long long ph[4] = {0, 0, 0, 0}, tc0 = 0;
    for (int t = 0; t < p.T; ++t) {
        if (probe) tc0 = clock64();
        // ---- prefetch this step's input-projection gates (independent of the barrier) ----
        float xgv[PAIRS][4];
        float skv[PAIRS];
#pragma unroll
        for (int pi = 0; pi < PAIRS; ++pi) {
            int idx = tid + pi * LSTM_WARPS * 32;
            int b = idx % LSTM_BT, u = idx / LSTM_BT;
            skv[pi] = (p.skip && idx < LSTM_BT * U && b < p.B) ? __ldg(p.skip + ((size_t)b * p.T + t) * H + j0 + u) : 0.f;
#pragma unroll
            for (int g = 0; g < 4; ++g)
                xgv[pi][g] = (idx < LSTM_BT * U && b < p.B)
                                 ? __ldg(p.xg + ((size_t)b * p.T + t) * (4 * H) + (size_t)g * H + j0 + u)
                                 : 0.f;
        }
        // ---- W_hh tiles do not depend on the barrier: put the first LSTM_D-1 of them in flight now ----
        auto issue_w = [&](int sub) {
            float* wsm = my_stage + (sub % LSTM_D) * STAGE_F + LSTM_KS * LSTM_HP;
            const float* wg = wsrc + (size_t)(k_begin + sub * LSTM_KS) * R;
#pragma unroll
            for (int i = lane; i < LSTM_KS * R / 4; i += 32) {
                int kr = i / (R / 4), c4 = i % (R / 4);
                cp_async16(wsm + kr * WP + c4 * 4, wg + kr * R + c4 * 4);
            }
        };
#pragma unroll
        for (int s0 = 0; s0 < LSTM_D - 1; ++s0) {
            if (s0 < nsub) issue_w(s0);
            cp_async_commit();
        }
        // ---- wait until every CTA has published h_{t-1} ----
        if (t > 0) {
            if (tid == 0) {
                unsigned target = (unsigned)p.G * (unsigned)t;
                unsigned v;
                do {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p.bar));
                } while (v < target);
            }
            __syncthreads();
        }
        const float* hprev = p.hT + (size_t)((t + 1) & 1) * H * LSTM_BT;  // parity of t-1
        if (probe) { long long n = clock64(); ph[0] += n - tc0; tc0 = n; }

        float acc[MT][NTL][4];
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int j = 0; j < NTL; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

        auto issue_h = [&](int sub) {
            float* hs = my_stage + (sub % LSTM_D) * STAGE_F;
            const float* hg = hprev + (size_t)(k_begin + sub * LSTM_KS) * LSTM_BT;
#pragma unroll
            for (int i = lane; i < LSTM_KS * LSTM_BT / 4; i += 32) {
                int kr = i / (LSTM_BT / 4), c4 = i % (LSTM_BT / 4);
                cp_async16(hs + kr * LSTM_HP + c4 * 4, hg + kr * LSTM_BT + c4 * 4);
            }
        };
#pragma unroll
        for (int s0 = 0; s0 < LSTM_D - 1; ++s0) {
            if (s0 < nsub) issue_h(s0);
            cp_async_commit();
        }
        // group order: W0..W(D-2), h0..h(D-2), [W+h](D-1), ... ; tile `sub` is complete once at most
        // D-1 younger groups are pending (an empty group is committed when nothing is left to issue)
        for (int sub = 0; sub < nsub; ++sub) {
            const int nxt = sub + LSTM_D - 1;
            if (nxt < nsub) { issue_w(nxt); issue_h(nxt); }
            cp_async_commit();
            cp_async_wait<LSTM_D - 1>();
            __syncwarp();
            const float* hs = my_stage + (sub % LSTM_D) * STAGE_F;
            const float* wsm = hs + LSTM_KS * LSTM_HP;
            if constexpr (BF16) {
                // one k16 step per sub-chunk.  B fragments: b0 = h[2t..2t+1][n0+g], b1 = h[2t+8..2t+9][n0+g]
                uint32_t bh[NTL][2], bl[NTL][2];
#pragma unroll
                for (int j = 0; j < NTL; ++j) {
                    const float* hp = hs + (2 * ft) * LSTM_HP + j * 8 + fg;
                    bf16_split2(hp[0], hp[LSTM_HP], bh[j][0], bl[j][0]);
                    bf16_split2(hp[8 * LSTM_HP], hp[9 * LSTM_HP], bh[j][1], bl[j][1]);
                }
                const uint32_t* wh = reinterpret_cast<const uint32_t*>(wsm);   // rows 0..7: hi k-pairs, 8..15: lo
#pragma unroll
                for (int i = 0; i < MT; ++i) {
                    // A fragments: a0 = (g, k 2t..), a1 = (g+8, k 2t..), a2 = (g, k 2t+8..), a3 = (g+8, k 2t+8..)
                    uint32_t ah[4], al[4];
                    ah[0] = wh[ft * WP + i * 16 + fg];           ah[1] = wh[ft * WP + i * 16 + fg + 8];
                    ah[2] = wh[(ft + 4) * WP + i * 16 + fg];     ah[3] = wh[(ft + 4) * WP + i * 16 + fg + 8];
                    al[0] = wh[(8 + ft) * WP + i * 16 + fg];     al[1] = wh[(8 + ft) * WP + i * 16 + fg + 8];
                    al[2] = wh[(12 + ft) * WP + i * 16 + fg];    al[3] = wh[(12 + ft) * WP + i * 16 + fg + 8];
#pragma unroll
                    for (int j = 0; j < NTL; ++j) {
                        mma_bf16_16x8x16(acc[i][j], al, bh[j]);    // small terms first
                        mma_bf16_16x8x16(acc[i][j], ah, bl[j]);
                        mma_bf16_16x8x16(acc[i][j], ah, bh[j]);
                    }
                }
            } else {
#pragma unroll
            for (int ks = 0; ks < LSTM_KS / 8; ++ks) {
                const int k0 = ks * 8;
                // B fragments: h[k][b], b0 = (k0+ft, n0+fg), b1 = (k0+ft+4, n0+fg); hi/lo split in registers
                float bh[NTL][2], bl[NTL][2];
#pragma unroll
                for (int j = 0; j < NTL; ++j) {
                    float v0 = hs[(k0 + ft) * LSTM_HP + j * 8 + fg];
                    float v1 = hs[(k0 + ft + 4) * LSTM_HP + j * 8 + fg];
                    bh[j][0] = tf32_rn(v0); bl[j][0] = tf32_rn(v0 - bh[j][0]);
                    bh[j][1] = tf32_rn(v1); bl[j][1] = tf32_rn(v1 - bh[j][1]);
                }
#pragma unroll
                for (int i = 0; i < MT; ++i) {
                    // A fragments: W[r][k] staged as wsm[k][r]; a0=(g,t) a1=(g+8,t) a2=(g,t+4) a3=(g+8,t+4)
                    float ah[4], al[4];
                    float w0 = wsm[(k0 + ft) * WP + i * 16 + fg];
                    float w1 = wsm[(k0 + ft) * WP + i * 16 + fg + 8];
                    float w2 = wsm[(k0 + ft + 4) * WP + i * 16 + fg];
                    float w3 = wsm[(k0 + ft + 4) * WP + i * 16 + fg + 8];
                    ah[0] = tf32_rn(w0); al[0] = tf32_rn(w0 - ah[0]);
                    ah[1] = tf32_rn(w1); al[1] = tf32_rn(w1 - ah[1]);
                    ah[2] = tf32_rn(w2); al[2] = tf32_rn(w2 - ah[2]);
                    ah[3] = tf32_rn(w3); al[3] = tf32_rn(w3 - ah[3]);
#pragma unroll
                    for (int j = 0; j < NTL; ++j) {
                        mma_tf32_16x8x8(acc[i][j], al, bh[j]);     // small terms first
                        mma_tf32_16x8x8(acc[i][j], ah, bl[j]);
                        mma_tf32_16x8x8(acc[i][j], ah, bh[j]);
                    }
                }
            }
            }
            __syncwarp();   // everyone done with this stage before it is refilled
        }
        if (probe) { long long n = clock64(); ph[1] += n - tc0; tc0 = n; }
        // ---- cross-warp reduction through shared memory: c0=(g,2t) c1=(g,2t+1) c2=(g+8,2t) c3=(g+8,2t+1) ----
        float* myred = my_stage;   // aliases this warp's own (fully consumed) stage buffers
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int j = 0; j < NTL; ++j) {
                const int r0 = i * 16 + fg, b0 = j * 8 + 2 * ft;
                myred[b0 * RP + r0] = acc[i][j][0];
                myred[(b0 + 1) * RP + r0] = acc[i][j][1];
                myred[b0 * RP + r0 + 8] = acc[i][j][2];
                myred[(b0 + 1) * RP + r0 + 8] = acc[i][j][3];
            }
        __syncthreads();

        float* hcur = p.hT + (size_t)(t & 1) * H * LSTM_BT;
#pragma unroll
        for (int pi = 0; pi < PAIRS; ++pi) {
            int idx = tid + pi * LSTM_WARPS * 32;
            if (idx >= LSTM_BT * U) break;
            int b = idx % LSTM_BT, u = idx / LSTM_BT;   // consecutive threads -> consecutive b (hT row)
            float g4[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                float s = 0.f;
#pragma unroll
                for (int w = 0; w < LSTM_WARPS; ++w) s += stage_base[w * LSTM_D * STAGE_F + b * RP + g * U + u];
                g4[g] = s + xgv[pi][g];
            }
            float ig = sigmoid_f(g4[0]), fg = sigmoid_f(g4[1]), gg = tanhf(g4[2]), og = sigmoid_f(g4[3]);
            float c = fg * cstate[b * U + u] + ig * gg;
            cstate[b * U + u] = c;
            float h = og * tanhf(c);
            hcur[(size_t)(j0 + u) * LSTM_BT + b] = h;
            if (b < p.B) {
                size_t o = ((size_t)b * p.T + t) * H + j0 + u;
                p.y[o] = h + skv[pi];
            }
        }
        if (probe) { long long n = clock64(); ph[2] += n - tc0; tc0 = n; }
        // ---- publish: CTA barrier orders every thread's h stores before thread 0, whose gpu-scope
        // fence is cumulative, then one release-arrive on the grid counter ----
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(p.bar, 1u);
        }
        if (probe) { long long n = clock64(); ph[3] += n - tc0; }
    }
    if (probe) { for (int i = 0; i < 4; ++i) g_lstm_phase_clock[i] = ph[i]; }
}

cudaError_t lstm_read_phase_clocks(long long* out4) { return cudaMemcpyFromSymbol(out4, g_lstm_phase_clock, sizeof(long long) * 4); }

int lstm_units_per_cta(int H) {
    if (H % 12 == 0 && H / 12 <= 132 && (H / LSTM_WARPS) % LSTM_KS == 0) return 12;
    if (H % 8 == 0 && H / 8 <= 132 && (H / LSTM_WARPS) % LSTM_KS == 0) return 8;
    return 0;
}

template <int U, bool BF16>
static cudaError_t launch_u(const LstmParams& p, cudaStream_t st) {
    constexpr int R = 4 * U;
    size_t smem = sizeof(float) * (LSTM_WARPS * LstmDepth<U>::D * LSTM_KS * (LstmHP<BF16>::V + R + 8) + LSTM_BT * U);
    cudaError_t e = cudaFuncSetAttribute(lstm_rec_kernel<U, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(p.bar, 0, sizeof(unsigned int), st);
    if (e != cudaSuccess) return e;
    // h_{-1} = 0 lives in parity slot 1
    e = cudaMemsetAsync(p.hT + (size_t)p.H * LSTM_BT, 0, sizeof(float) * p.H * LSTM_BT, st);
    if (e != cudaSuccess) return e;
    LstmParams pp = p;
    void* args[] = {&pp};
    return cudaLaunchCooperativeKernel((void*)lstm_rec_kernel<U, BF16>, dim3(p.G), dim3(LSTM_WARPS * 32), args, smem, st);
}

cudaError_t launch_lstm_layer(const LstmParams& p, cudaStream_t st) {
    if (p.B > LSTM_BT || p.B <= 0) return cudaErrorInvalidValue;
    if (p.bf16 && !p.whh_p16) return cudaErrorInvalidValue;
    if (p.U == 8) return p.bf16 ? launch_u<8, true>(p, st) : launch_u<8, false>(p, st);
    if (p.U == 12) return p.bf16 ? launch_u<12, true>(p, st) : launch_u<12, false>(p, st);
    return cudaErrorInvalidValue;
}

}  // namespace fac
