// Persistent LSTM recurrence, second generation (SLSTM: dac/model/encodec.py:272-288 -> nn.LSTM(C, C, 2)).
//
// Same decomposition as lstm.cu (input projections = one GEMM; this kernel = the serial chain
// gates_t = xg_t + h_{t-1} W_hh^T; one cooperative launch per layer, CTA c owns hidden units [c*U, c*U+U), cell state in
// shared memory, h_t exchanged through L2 with one grid barrier per step), rebuilt around what the round-1 profile showed
// (12.9 ms per step of the benchmark, 15 %): W_hh re-streamed from L2 every step, fp32 h split in registers inside the
// K loop, TF32 m16n8k8 tiles upstream.
//
//   * W_hh stays RESIDENT in shared memory for the whole sequence, pre-split offline into fp16 words (two consecutive k per
//     32-bit word = one mma.sync m16n8k16 A-fragment register), XOR-swizzled so the fragment loads are conflict-free
//     without padding: 128 KB (H = 1024: hi + scaled lo) / 144 KB (H = 1536: hi only) per CTA.
//   * h_t is PUBLISHED already split into fp16 words in the B-fragment layout ([k pair][batch], swizzled): the K loop is
//     cp.async -> LDS -> MMA, no conversions.
//   * PASS3 = true (upstream of the VQ): a*b ~= a_hi*b_hi + (a_hi*b_lo' + a_lo'*b_hi) * 2^-11 with fp16 hi and lo' =
//     rn_f16((x - hi) * 2^11): 22 mantissa bits like the TF32 pair, half the MMA instructions (K = 16); the scaled cross
//     terms have their own fp32 accumulators.
//   * PASS3 = false (downstream of the VQ): ONE fp16 pass.  Measured on the oracle (scripts/cpu_lstm_precision.py): rounding
//     W_hh and h of the decoder's LSTM to fp16 moves the reconstructed waveform by 1.9e-7 RMS (bar 1e-4; bf16 hi+lo kept
//     as "decoder_lstm_fp16" = 0).
//
// A step needs H/16 k-steps x passes = 96-192 dependent MMAs per CTA on a 32-row tile: warp-level mma.sync keeps that
// latency chain short; an asynchronous warpgroup MMA pipeline only pays off on tiles far larger than one step.
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace fac {

__device__ long long g_lstm2_phase_clock[4];

namespace {
constexpr int L2_BT = 32;       // batch tile
constexpr int L2_WARPS = 8;
// cp.async ring depth per warp (stages of one k16 sub-chunk of h): 4 x 2 KB (hi + lo') upstream, 8 x 1 KB downstream
template <bool PASS3> struct L2Depth { static constexpr int D = PASS3 ? 4 : 8; };

__device__ __forceinline__ void mma_f16_16x8x16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void cp16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
}  // namespace

// swizzles shared by the host packer, the publisher and the fragment loads
__host__ __device__ __forceinline__ int lstm2_swz_w(int k2, int R) { return R == 32 ? ((k2 & 3) << 3) : (((k2 >> 1) & 1) << 3); }
__host__ __device__ __forceinline__ int lstm2_swz_h(int kp) { return (kp & 3) << 3; }

// h exchange buffer: [2 parities][PL planes][H/2 k pairs][32] words; PL = 2 (hi, lo') when PASS3 else 1.  LENS: the per-lane
// step counts of LstmLaneLens apply (LstmLenParams); without them the kernel is the one it always was.  REV (with LENS): the
// reverse direction of a bidirectional layer -- step s of lane b reads and writes frame len[b] - 1 - s, so every lane starts
// at its own last frame.
struct LstmLenParams : LstmParams { LstmLaneLens lens; };
template <int U, bool PASS3, bool LENS, bool REV = false>
__global__ void __launch_bounds__(L2_WARPS * 32, 1) lstm_rec2_kernel(std::conditional_t<LENS, LstmLenParams, LstmParams> p) {
    static_assert(!REV || LENS, "the reverse direction needs the lane lengths");
    constexpr int R = 4 * U;
    constexpr int RP = R + 1;
    constexpr int MT = R / 16, NTL = L2_BT / 8;
    constexpr int PL = PASS3 ? 2 : 1;
    constexpr int L2_DEPTH = L2Depth<PASS3>::D;
    constexpr int STAGE_W = PL * 8 * L2_BT;                    // words per stage (one k16 sub-chunk of h): 256 / 512
    static_assert(L2_DEPTH * STAGE_W >= L2_BT * RP, "reduction buffer must fit in a warp's own stage memory");
    extern __shared__ __align__(16) uint32_t smem2[];
    const int H = p.H;
    const int nsub_all = H / 16;
    uint32_t* wres = smem2;                                                      // [H/16][PL][8][R] resident W_hh slice
    uint32_t* stage_base = wres + (size_t)nsub_all * PL * 8 * R;                 // [8 warps][L2_DEPTH][STAGE_W]
    float* cstate = reinterpret_cast<float*>(stage_base + L2_WARPS * L2_DEPTH * STAGE_W);   // [32][U]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x;
    const int j0 = cta * U;
    const int nsub = nsub_all / L2_WARPS;          // k16 sub-chunks per warp
    const int sub0 = warp * nsub;
    const int fg = lane >> 2, ft = lane & 3;

    // ---- one-time: W_hh slice -> shared memory (linear copy: the swizzle is baked into the packed layout) ----
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.whh_p2 + (size_t)cta * nsub_all * PL * 8 * R);
        uint4* dst = reinterpret_cast<uint4*>(wres);
        const int n16 = nsub_all * PL * 8 * R / 4;
        for (int i = tid; i < n16; i += blockDim.x) dst[i] = __ldg(src + i);
    }
    // cell state: zero (nn.LSTM default) or carried over from the previous chunk of a stream (state_c: [G][32][U])
    for (int i = tid; i < L2_BT * U; i += blockDim.x) cstate[i] = p.state_c ? p.state_c[(size_t)cta * L2_BT * U + i] : 0.f;
    __syncthreads();

    uint32_t* my_stage = stage_base + warp * L2_DEPTH * STAGE_W;
    const size_t plane_words = (size_t)(H / 2) * L2_BT;       // one plane of one parity
    constexpr int PAIRS = (L2_BT * U + L2_WARPS * 32 - 1) / (L2_WARPS * 32);
    const bool probe = (cta == 0 && tid == 0);
    long long ph[4] = {0, 0, 0, 0}, tc0 = 0;

    for (int t = 0; t < p.T; ++t) {
        if (probe) tc0 = clock64();
        // ---- this step's input-projection gates (independent of the barrier) ----
        float xgv[PAIRS][4];
        float skv[PAIRS];
#pragma unroll
        for (int pi = 0; pi < PAIRS; ++pi) {
            int idx = tid + pi * L2_WARPS * 32;
            int b = idx % L2_BT, u = idx / L2_BT;
            int tx = t;
            if constexpr (REV) tx = (b < p.B ? p.lens.len[b] : 0) - 1 - t;
            const bool in = idx < L2_BT * U && b < p.B && tx >= 0;
            skv[pi] = (p.skip && in) ? __ldg(p.skip + ((size_t)b * p.T + tx) * H + j0 + u) : 0.f;
#pragma unroll
            for (int g = 0; g < 4; ++g)
                xgv[pi][g] = in ? __ldg(p.xg + ((size_t)b * p.T + tx) * (4 * H) + (size_t)g * H + j0 + u) : 0.f;
        }
        // ---- wait until every CTA has published h_{t-1} ----
        if (t > 0) {
            if (tid == 0) {
                unsigned target = (unsigned)p.G * (unsigned)t;
                unsigned v;
                long long w0 = clock64();
                do {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p.bar));
                    if (v < target && clock64() - w0 > 4000000000LL) __trap();
                } while (v < target);
            }
            __syncthreads();
        }
        const uint32_t* hprev = p.h16 + (size_t)((t + 1) & 1) * PL * plane_words;   // parity of t-1
        if (probe) { long long n = clock64(); ph[0] += n - tc0; tc0 = n; }

        float acc0[MT][NTL][4];
        float acc1[PASS3 ? MT : 1][PASS3 ? NTL : 1][4];
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int j = 0; j < NTL; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) { acc0[i][j][e] = 0.f; if (PASS3) acc1[i][j][e] = 0.f; }

        // stage s of the ring <- sub-chunk `sub` of this warp's K slice: 8 k pairs x 32 batch words per plane (1 KB each)
        auto issue_h = [&](int sub) {
            uint32_t* hs = my_stage + (sub % L2_DEPTH) * STAGE_W;
#pragma unroll
            for (int pl = 0; pl < PL; ++pl) {
                const uint32_t* hg = hprev + pl * plane_words + (size_t)(sub0 + sub) * 8 * L2_BT;
#pragma unroll
                for (int i = lane; i < 8 * L2_BT / 4; i += 32) cp16(hs + pl * 8 * L2_BT + i * 4, hg + i * 4);
            }
        };
#pragma unroll
        for (int s0 = 0; s0 < L2_DEPTH - 1; ++s0) {
            if (s0 < nsub) issue_h(s0);
            cp_commit();
        }
        for (int sub = 0; sub < nsub; ++sub) {
            const int nxt = sub + L2_DEPTH - 1;
            if (nxt < nsub) issue_h(nxt);
            cp_commit();
            cp_wait<L2_DEPTH - 1>();
            __syncwarp();
            const uint32_t* hs = my_stage + (sub % L2_DEPTH) * STAGE_W;
            const uint32_t* wh = wres + (size_t)(sub0 + sub) * PL * 8 * R;
            // B fragments: b0 = word(k pair ft, n), b1 = word(k pair ft + 4, n); columns swizzled by the k pair
            uint32_t bh[NTL][2], bl[PASS3 ? NTL : 1][2];
#pragma unroll
            for (int j = 0; j < NTL; ++j) {
                const int c0 = (j * 8 + fg) ^ lstm2_swz_h(ft);
                bh[j][0] = hs[ft * L2_BT + c0];
                bh[j][1] = hs[(ft + 4) * L2_BT + c0];
                if (PASS3) {
                    bl[j][0] = hs[8 * L2_BT + ft * L2_BT + c0];
                    bl[j][1] = hs[8 * L2_BT + (ft + 4) * L2_BT + c0];
                }
            }
            const int sw = lstm2_swz_w(ft, R);
#pragma unroll
            for (int i = 0; i < MT; ++i) {
                // A fragments: a0 = (row g, k pair ft), a1 = (row g+8, ft), a2 = (row g, ft+4), a3 = (row g+8, ft+4)
                uint32_t ah[4], al[4];
                const int r0 = (i * 16 + fg) ^ sw, r1 = (i * 16 + fg + 8) ^ sw;
                ah[0] = wh[ft * R + r0];        ah[1] = wh[ft * R + r1];
                ah[2] = wh[(ft + 4) * R + r0];  ah[3] = wh[(ft + 4) * R + r1];
                if (PASS3) {
                    al[0] = wh[8 * R + ft * R + r0];        al[1] = wh[8 * R + ft * R + r1];
                    al[2] = wh[8 * R + (ft + 4) * R + r0];  al[3] = wh[8 * R + (ft + 4) * R + r1];
                }
#pragma unroll
                for (int j = 0; j < NTL; ++j) {
                    mma_f16_16x8x16(acc0[i][j], ah, bh[j]);
                    if (PASS3) {
                        mma_f16_16x8x16(acc1[i][j], ah, bl[j]);
                        mma_f16_16x8x16(acc1[i][j], al, bh[j]);
                    }
                }
            }
            __syncwarp();
        }
        if (probe) { long long n = clock64(); ph[1] += n - tc0; tc0 = n; }
        // ---- cross-warp reduction through shared memory (aliases this warp's own, fully consumed, stage buffers) ----
        float* myred = reinterpret_cast<float*>(my_stage);
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
            for (int j = 0; j < NTL; ++j) {
                const int r0 = i * 16 + fg, b0 = j * 8 + 2 * ft;
                float v0 = acc0[i][j][0], v1 = acc0[i][j][1], v2 = acc0[i][j][2], v3 = acc0[i][j][3];
                if (PASS3) {
                    v0 = fmaf(acc1[i][j][0], 1.0f / 2048.0f, v0); v1 = fmaf(acc1[i][j][1], 1.0f / 2048.0f, v1);
                    v2 = fmaf(acc1[i][j][2], 1.0f / 2048.0f, v2); v3 = fmaf(acc1[i][j][3], 1.0f / 2048.0f, v3);
                }
                myred[b0 * RP + r0] = v0;
                myred[(b0 + 1) * RP + r0] = v1;
                myred[b0 * RP + r0 + 8] = v2;
                myred[(b0 + 1) * RP + r0 + 8] = v3;
            }
        __syncthreads();

        __half* hcur = reinterpret_cast<__half*>(p.h16 + (size_t)(t & 1) * PL * plane_words);
#pragma unroll
        for (int pi = 0; pi < PAIRS; ++pi) {
            int idx = tid + pi * L2_WARPS * 32;
            if (idx >= L2_BT * U) break;
            int b = idx % L2_BT, u = idx / L2_BT;
            float g4[4];
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                float s = 0.f;
#pragma unroll
                for (int w = 0; w < L2_WARPS; ++w)
                    s += reinterpret_cast<const float*>(stage_base + w * L2_DEPTH * STAGE_W)[b * RP + g * U + u];
                g4[g] = s + xgv[pi][g];
            }
            float ig = sigmoid_f(g4[0]), fgt = sigmoid_f(g4[1]), gg = tanhf(g4[2]), og = sigmoid_f(g4[3]);
            float c = fgt * cstate[b * U + u] + ig * gg;
            if constexpr (LENS) {
                // the line above spelled out as the no-length kernel compiles it (ig * gg fused onto fgt * c), so that a
                // lane's bits do not depend on which of the two instantiations runs it
                c = __fmaf_rn(ig, gg, __fmul_rn(fgt, cstate[b * U + u]));
                if (t >= p.lens.len[b]) {
                    // past the lane's length: keep c and re-publish h_{t-1} (this thread's own unit, written by no other
                    // CTA); the output row is a finite don't-care
                    const int k = j0 + u, kp = k >> 1;
                    const size_t widx = (size_t)kp * L2_BT + (size_t)(b ^ lstm2_swz_h(kp));
                    const __half* hp = reinterpret_cast<const __half*>(hprev);
                    hcur[widx * 2 + (k & 1)] = hp[widx * 2 + (k & 1)];
                    if (PASS3) hcur[(plane_words + widx) * 2 + (k & 1)] = hp[(plane_words + widx) * 2 + (k & 1)];
                    if (b < p.B) p.y[((size_t)b * p.T + t) * H + j0 + u] = skv[pi];
                    continue;
                }
            }
            cstate[b * U + u] = c;
            float h = og * tanhf(c);
            // publish h_t pre-split: word (k pair, batch) holds units 2kp (low half) and 2kp+1
            const int k = j0 + u, kp = k >> 1;
            const size_t widx = (size_t)kp * L2_BT + (size_t)(b ^ lstm2_swz_h(kp));
            const __half hh = __float2half_rn(h);
            hcur[widx * 2 + (k & 1)] = hh;
            if (PASS3) hcur[(plane_words + widx) * 2 + (k & 1)] = __float2half_rn((h - __half2float(hh)) * 2048.0f);
            if (b < p.B) {
                int ty = t;
                if constexpr (REV) ty = p.lens.len[b] - 1 - t;
                size_t o = ((size_t)b * p.T + ty) * H + j0 + u;
                p.y[o] = h + skv[pi];
            }
        }
        if (probe) { long long n = clock64(); ph[2] += n - tc0; tc0 = n; }
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(p.bar, 1u);
        }
        if (probe) { long long n = clock64(); ph[3] += n - tc0; }
    }
    if (p.state_c) {
        __syncthreads();
        for (int i = tid; i < L2_BT * U; i += blockDim.x) p.state_c[(size_t)cta * L2_BT * U + i] = cstate[i];
    }
    if (probe) { for (int i = 0; i < 4; ++i) g_lstm2_phase_clock[i] = ph[i]; }
}

cudaError_t lstm2_read_phase_clocks(long long* out4) { return cudaMemcpyFromSymbol(out4, g_lstm2_phase_clock, sizeof(long long) * 4); }

// Host: nn.LSTM weight_hh [4H][H] (gate order i,f,g,o) -> [G][H/16][planes][8 k pairs][R] fp16-pair words, column of row r
// of k pair k2 = r ^ lstm2_swz_w(k2, R); planes = {hi, lo' = rn_f16((w - hi) * 2^11)} when pass3 else {hi}.
size_t lstm2_pack_words(int H, int U, int pass3) { return (size_t)(H / U) * (H / 16) * (pass3 ? 2 : 1) * 8 * (4 * U); }
void lstm2_pack(const float* whh, int H, int U, int pass3, uint32_t* out) {
    const int G = H / U, R = 4 * U, PL = pass3 ? 2 : 1;
    auto bits = [](__half v) { uint16_t b; memcpy(&b, &v, 2); return (uint32_t)b; };
    for (int cta = 0; cta < G; ++cta)
        for (int sub = 0; sub < H / 16; ++sub)
            for (int k2 = 0; k2 < 8; ++k2)
                for (int r = 0; r < R; ++r) {
                    const int g = r / U, u = r % U;
                    const float* wrow = &whh[((size_t)g * H + cta * U + u) * H + sub * 16 + 2 * k2];
                    const __half h0 = __float2half_rn(wrow[0]), h1 = __float2half_rn(wrow[1]);
                    const size_t base = (((size_t)cta * (H / 16) + sub) * PL) * 8 * R;
                    const int col = r ^ lstm2_swz_w(k2, R);
                    out[base + (size_t)k2 * R + col] = bits(h0) | (bits(h1) << 16);
                    if (pass3) {
                        const __half l0 = __float2half_rn((wrow[0] - __half2float(h0)) * 2048.0f);
                        const __half l1 = __float2half_rn((wrow[1] - __half2float(h1)) * 2048.0f);
                        out[base + (size_t)(8 + k2) * R + col] = bits(l0) | (bits(l1) << 16);
                    }
                }
}

size_t lstm2_smem_bytes(int H, int U, int pass3) {
    const int R = 4 * U, PL = pass3 ? 2 : 1;
    const int depth = pass3 ? 4 : 8;
    return sizeof(uint32_t) * ((size_t)(H / 16) * PL * 8 * R + (size_t)L2_WARPS * depth * PL * 8 * L2_BT) + sizeof(float) * L2_BT * U;
}

// state_h: [planes][H/2 k pairs][32] words, the layout the kernel publishes h in; state_c: [G][32][U] (per-CTA cell state)
void lstm2_state_sizes(int H, int U, int pass3, size_t* h_words, size_t* c_floats) {
    *h_words = (size_t)(pass3 ? 2 : 1) * (H / 2) * L2_BT;
    *c_floats = (size_t)(H / U) * L2_BT * U;
}

// Position of word j of lane b's carry: h word (plane pl, k pair kp) at pl * H/2 * 32 + kp * 32 + (b ^ lstm2_swz_h(kp)), then
// the cell state of unit k (CTA k / U) at h_words + (k / U) * 32 * U + b * U + k % U.
__host__ __device__ __forceinline__ long long lstm2_lane_word(int H, int U, int pl_count, int b, int j) {
    const int hw = pl_count * (H / 2);
    if (j < hw) {
        const int pl = j / (H / 2), kp = j % (H / 2);
        return (long long)pl * (H / 2) * L2_BT + (long long)kp * L2_BT + (b ^ lstm2_swz_h(kp));
    }
    const int k = j - hw;
    return (long long)hw * L2_BT + (long long)(k / U) * L2_BT * U + (long long)b * U + k % U;
}

void lstm2_lane_map(int H, int U, int pass3, int b, long long* pos) {
    const int PL = pass3 ? 2 : 1;
    for (int j = 0; j < PL * (H / 2) + H; ++j) pos[j] = lstm2_lane_word(H, U, PL, b, j);
}

__global__ void lstm2_lane_carry_kernel(LaneCarryParams p) {
    const int b = blockIdx.y;
    if (b >= p.n) return;
    const int PL = p.pass3 ? 2 : 1, words = PL * (p.H / 2) + p.H;
    const long long hw = (long long)PL * (p.H / 2) * L2_BT;
    uint32_t* slot = p.slot[b];
    uint32_t* cw = reinterpret_cast<uint32_t*>(p.state_c);
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < words; j += gridDim.x * blockDim.x) {
        const long long pos = lstm2_lane_word(p.H, p.U, PL, b, j);
        uint32_t* w = pos < hw ? p.state_h + pos : cw + (pos - hw);
        if (p.to_lanes) *w = slot[j];
        else slot[j] = *w;
    }
}

cudaError_t launch_lstm2_lane_carry(const LaneCarryParams& p, cudaStream_t st) {
    if (p.n <= 0) return cudaSuccess;
    if (p.n > L2_BT || p.U <= 0 || p.H % p.U != 0) return cudaErrorInvalidValue;
    lstm2_lane_carry_kernel<<<dim3(8, p.n), 256, 0, st>>>(p);
    return cudaGetLastError();
}

template <int U, bool PASS3, bool LENS, bool REV = false>
static cudaError_t launch2_u(const LstmParams& p, const LstmLaneLens* lens, cudaStream_t st) {
    const size_t smem = lstm2_smem_bytes(p.H, U, PASS3 ? 1 : 0);
    if (smem > 227 * 1024) return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(lstm_rec2_kernel<U, PASS3, LENS, REV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(p.bar, 0, sizeof(unsigned int), st);
    if (e != cudaSuccess) return e;
    // h_{-1} = 0 lives in parity slot 1 (all planes)
    const size_t plane_words = (size_t)(p.H / 2) * L2_BT;
    const int PL = PASS3 ? 2 : 1;
    // ... or the carried-over h of a stream (state_h: [planes][H/2][32] words, the layout the kernel publishes)
    if (p.state_h) e = cudaMemcpyAsync(p.h16 + (size_t)PL * plane_words, p.state_h, sizeof(uint32_t) * PL * plane_words, cudaMemcpyDeviceToDevice, st);
    else e = cudaMemsetAsync(p.h16 + (size_t)PL * plane_words, 0, sizeof(uint32_t) * PL * plane_words, st);
    if (e != cudaSuccess) return e;
    std::conditional_t<LENS, LstmLenParams, LstmParams> pp;
    static_cast<LstmParams&>(pp) = p;
    if constexpr (LENS) pp.lens = *lens;
    void* args[] = {&pp};
    e = cudaLaunchCooperativeKernel((void*)lstm_rec2_kernel<U, PASS3, LENS, REV>, dim3(p.G), dim3(L2_WARPS * 32), args, smem, st);
    if (e != cudaSuccess) return e;
    // h_{T-1} was published into parity slot (T-1) & 1
    if (p.state_h) e = cudaMemcpyAsync(p.state_h, p.h16 + (size_t)((p.T - 1) & 1) * PL * plane_words, sizeof(uint32_t) * PL * plane_words, cudaMemcpyDeviceToDevice, st);
    return e;
}

cudaError_t launch_lstm2_layer(const LstmParams& p, cudaStream_t st, const LstmLaneLens* lens, bool reverse) {
    if (p.B > L2_BT || p.B <= 0 || !p.whh_p2 || !p.h16) return cudaErrorInvalidValue;
    if ((p.H / 16) % L2_WARPS != 0) return cudaErrorInvalidValue;
    if (reverse) {   // the fp32-faithful class (JDCNet's BiLSTM), no carried stream state
        if (!lens || !p.pass3 || p.state_h || p.state_c) return cudaErrorInvalidValue;
        for (int b = 0; b < p.B; ++b)
            if (lens->len[b] < 0 || lens->len[b] > p.T) return cudaErrorInvalidValue;
        if (p.U == 8) return launch2_u<8, true, true, true>(p, lens, st);
        if (p.U == 12) return launch2_u<12, true, true, true>(p, lens, st);
        return cudaErrorInvalidValue;
    }
    if (lens) {   // the one-pass class (the decoder's LSTM) only
        if (p.pass3) return cudaErrorInvalidValue;
        if (p.U == 8) return launch2_u<8, false, true>(p, lens, st);
        if (p.U == 12) return launch2_u<12, false, true>(p, lens, st);
        return cudaErrorInvalidValue;
    }
    if (p.U == 8) return p.pass3 ? launch2_u<8, true, false>(p, lens, st) : launch2_u<8, false, false>(p, lens, st);
    if (p.U == 12) return p.pass3 ? launch2_u<12, true, false>(p, lens, st) : launch2_u<12, false, false>(p, lens, st);
    return cudaErrorInvalidValue;
}

}  // namespace fac
