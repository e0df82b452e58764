// Channels-last 1-D convolution on the Hopper tensor cores (wgmma, sm_90a), fp32-faithful.
//
// Same contract as conv_simt.cu (SConv1d / SConvTranspose1d / Linear call sites of the
// reference), restricted to stride-1 convs in "rows" (a strided down-conv with kernel 2s is a
// 2-tap conv over rows of s consecutive samples, see `vf`), Cin*vf % 16 == 0, Cout % 16 == 0.
//
//   D[t][co] = sum_tap sum_j  A[t - PLr + tap*dil][j] * W[tap][j][co]
//
// Precision: bit-exact VQ indices need fp32-faithful sums (SURVEY.md 0.5), so every product is
// formed as 3 MMAs over split operands (x = hi + lo):
//   a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi     (dropped term a_lo*b_lo ~ 2^-22 |ab|)
// Weights are split offline (tc_pack_blob); activations are split in-kernel.  Split classes:
//   TF32 pairs (k = 8 MMAs); bf16 pairs (k = 16) downstream of the VQ; ONE fp16 pass (g1f16: the k = 7 convs
//   downstream of the VQ); fp16 hi + 2^11-scaled fp16 lo (f16x2, promoted only).
// Promoted layers (upstream of the VQ, long K loops) accumulate each window of <= 48 chained MMAs in fresh
// registers and add it to an fp32 master accumulator, so the sum is not one long tensor-core accumulation chain.  The
// master lives in shared memory, so the window registers are the only accumulators and the promoted class fits the
// register budget of two resident CTAs per SM.
//
// CTA = two warpgroups over a tile of 128 rows x N channels (each warpgroup 64 rows) or 64 rows x N channels (each
// warpgroup N/2 channels).  A warpgroup spans at most 128 channels, except in the one-pass fp16 class: its tiles of the
// decoder's C = 768 conv7 (N = 256) and C = 192 fused unit (N = 192) are 128 rows with each warpgroup over all N channels
// (see tc_conv_plan).  Per step of `group` (1, 2 or 4) 16-channel chunks, 2-4 only on layers of 1-3 taps:
//   weights: one thread streams the chunk's pre-arranged [tap][hi|lo][k-piece][N][16 B] blob with ONE 1-D bulk copy
//            (cp.async.bulk, completion on an mbarrier) into a ring of 1-2 slots;
//   activations: all 256 threads load the UNION of the rows all taps need (rows + (K-1)*dil) once with 16-byte loads
//            (reflect / zero padding = index map, no padded copy), apply Snake, split into hi/lo and store them in a
//            no-swizzle K-major layout whose row pitch is a uniform 16 bytes, so each tap is just a descriptor
//            start-address offset of tap*dil rows (taps are never re-loaded or im2col'ed);
//   the next chunk's activations are produced while this chunk's wgmma run (double-buffered operand).
// Fused mode (a whole ResidualUnit, conv7 -> +b7 -> Snake -> 1x1 conv -> +b1 -> +x): GEMM 1's accumulators go through
// bias + Snake + split straight into a resident shared-memory operand for GEMM 2.  The promoted fp16 hi + scaled-lo class
// has it too (the encoder's C = 64 and C = 128 units, two CTAs per SM): GEMM 1 is the promoted conv7 with its windows,
// the split is split_store_f16's, and GEMM 2 runs the unfused 1x1's passes as one window, so the unit's output is the
// two-launch route's bit for bit without the conv7 output's round trip through global memory.  Its GEMM-2 operand
// takes the place of the master accumulator, which is dead after GEMM 1's last promotion.
// Epilogue from the accumulator registers: bias -> Snake/tanh/Mish -> residual -> 8-byte stores.
// Variants: tiles planned for two resident CTAs per SM (always tried for the promoted class; option "tc_occ2_maxn" for
// the others), and the transposed formulation of the promoted fp16 class (option "encoder_tt": weights as the wgmma A
// operand, time as wgmma N).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstring>
#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "conv_tc_common.cuh"
#include "kernels.h"

namespace fac {

namespace {

using namespace tc;

enum Prec { P_TF32 = 0, P_BF16 = 1, P_F16S = 2, P_F16X2 = 3, P_NONE = -1 };

template <int P> struct PrecT {
    static constexpr int KG = P == P_TF32 ? 4 : 2;           // 16-byte k-pieces per 16-channel chunk and plane
    static constexpr int planes = P == P_F16S ? 1 : 2;       // hi (+ lo)
    static constexpr int ksteps = P == P_TF32 ? 2 : 1;       // MMAs per chunk, tap and split pass
    static constexpr int kind = P == P_TF32 ? WG_TF32 : (P == P_BF16 ? WG_BF16 : WG_F16);
};

__host__ __device__ constexpr int prec_kg(int P) { return P == P_TF32 ? 4 : 2; }
__host__ __device__ constexpr int prec_planes(int P) { return P == P_F16S ? 1 : 2; }
// Shared-memory master accumulator of a promoted layer: the NI / 2 accumulator floats of every thread, float4 q of
// thread tid at q * kThreads + tid (lane-consecutive, so conflict-free).  A K loop of one window needs none.
__host__ __device__ constexpr uint32_t master_bytes(bool promoted, int nchunk, int promote_every, int ni) {
    return promoted && nchunk > promote_every ? (uint32_t)ni / 2 * 4 * kThreads : 0u;
}

template <int NI>
__device__ __forceinline__ void zero_acc(float (&a)[NI / 2]) {
#pragma unroll
    for (int i = 0; i < NI / 2; ++i) a[i] = 0.f;
}

// One operand pair (A rows x K-pieces, B channels x K-pieces) of one chunk: one wgmma per k-step over the warpgroup's
// whole width.  No runtime condition may guard these: ptxas then fences every wgmma with its own warpgroup.arrive and
// wait, and the chunk's MMAs run one after another instead of as one chained batch.
template <int P, int NI>
__device__ __forceinline__ void mma_pass(float (&acc)[NI / 2], uint32_t a_addr, uint32_t a_lbo, uint32_t b_addr,
                                         uint32_t b_lbo) {
#pragma unroll
    for (int ks = 0; ks < PrecT<P>::ksteps; ++ks)
        wgmma_ss<NI, PrecT<P>::kind>(acc, gdesc(a_addr + ks * 2 * a_lbo, a_lbo, 128), gdesc(b_addr + ks * 2 * b_lbo, b_lbo, 128));
}

struct Tile {
    int row0, col0, nw;       // this warpgroup's first tile row / channel, its channel width NW
    int warp, lane;
};

// Accumulator fragment of wgmma m64nNI: register 4j + 2h + e holds row 16*warp + lane/4 + 8h, column 8j + 2*(lane%4) + e.
// GROUP < NI cuts the unrolled loop into blocks of GROUP columns at a branch on the runtime width, never taken (the
// launcher picks NI == NW).  ptxas schedules each block on its own: the fused GEMM-1 epilogue (a Snake per element)
// takes 224 registers at NI = 128 as one block, and <= 128 in blocks of 32 columns.
template <int NI, int GROUP = NI, typename F>
__device__ __forceinline__ void for_each_pair(const Tile& tl, const float (&acc)[NI / 2], F&& f) {
#pragma unroll
    for (int j = 0; j < NI / 8; ++j) {
        if (j > 0 && (8 * j) % GROUP == 0 && 8 * j >= tl.nw) break;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = tl.row0 + 16 * tl.warp + (tl.lane >> 2) + 8 * h;
            const int col = tl.col0 + 8 * j + 2 * (tl.lane & 3);
            f(row, col, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

template <bool FAST>
__device__ __forceinline__ float act_out(int act, float v, float al, float ia) {
    if (act == ACT_SNAKE) return FAST ? fmaf(ia, sin2_mufu(al * v), v) : snake_fast(v, al, ia);
    if (act == ACT_TANH) return tanhf(v);
    if (act == ACT_MISH) return mish_f(v);
    return v;
}

// P1: split class of the layer's own GEMM; P2: of the fused GEMM 2 (P_NONE = not fused); NI: wgmma N, the warpgroup's
// whole channel width NW (NI / 2 accumulator registers per thread; NI <= 64 when promoted or MINB = 2, <= 256 in the
// one-pass fp16 class, else <= 128);
// MINB = 2: compiled for two resident CTAs per SM (<= 128 registers); the promoted class is only compiled so, and runs
// one CTA per SM when its plan needs more than half the shared memory;
// TT: transposed formulation -- the weights are the wgmma A operand (64 output channels per warpgroup) and time is the
// wgmma N dimension (NI = 64 time steps); the operand buffers and the weight blob are the same K-major layouts as the
// plain formulation.
// Grouping (p.group > 1, see tc_conv_plan) exists only in the instantiations that can plan it: not the one-pass fp16
// class, fused units or the transposed formulation, which keep the one-chunk K loop and producer.  The others run the
// grouped K loop at every G; they are register-bounded for two CTAs per SM at NI <= 128 (the grouped loop would take
// some past 128), so a plan within half the shared memory keeps two CTAs per SM.
template <int P1, int P2, bool TT>
constexpr bool groupable() { return P1 != P_F16S && P2 == P_NONE && !TT; }

// C2D: the 3x3 Conv2d of conv2d_tc_kernel over a channels-last [T][row2d][C] map, row2d = F + 2 (two zero frequency
// columns).  Flattened to rows, tap (dt, df) is the row offset dt * row2d + df from PLr = row2d + 1 rows back, so the
// operand holds BM + 2 row2d + 2 rows and each tap is again a descriptor start-address offset; the epilogue applies
// LeakyReLU(0.01) and writes the output's pad columns as zeros, so the output is the next layer's input layout.
template <int P1, int P2, bool PROMO, int NI, int MINB, bool TT, bool C2D>
__device__ __forceinline__ void conv_tc_body(const TcConvParams& p) {
    constexpr bool FUSED = P2 != P_NONE;
    constexpr bool GROUPABLE = groupable<P1, P2, TT>() && !C2D;
    static_assert(!C2D || (P1 == P_F16X2 && PROMO && !FUSED && !TT), "2-D taps: the promoted fp16 hi + scaled-lo class only");
    static_assert(!TT || (NI == 64 && !FUSED), "transposed tiles: <= 64 channels x 64 time steps per warpgroup");
    static_assert(NI % 16 == 0 && NI <= (PROMO || MINB == 2 ? 64 : (P1 == P_F16S ? 256 : 128)),
                  "accumulator registers: <= 64 / 128 columns (256 in the one-pass fp16 class at one CTA per SM)");
    constexpr bool F16X2 = P1 == P_F16X2;
    constexpr bool DEC = P1 == P_BF16 || P1 == P_F16S;      // downstream of the VQ: SFU-sine Snake class
    using T1 = PrecT<P1>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);

    const int tid = threadIdx.x, wg = tid >> 7;
    const int BM = 64 * p.MT;                               // MT = 2: warpgroups split rows; 1: they split channels
    const int N = p.N, NW = p.MT == 2 ? N : N / 2;
    Tile tl;
    tl.row0 = p.MT == 2 ? 64 * wg : 0;
    tl.col0 = p.MT == 2 ? 0 : wg * NW;
    tl.nw = NW;
    tl.warp = (tid >> 5) & 3;
    tl.lane = tid & 31;
    const int t0 = blockIdx.x * BM, ntile = blockIdx.y, b = blockIdx.z;
    const int Kr = p.Kr, dil = p.dil, Rpad = p.Rpad, nchunk = p.nchunk, S = p.stagesB;
    const int G = GROUPABLE ? p.group : 1;                   // chunks per GEMM-1 step: 1, 2 or 4
    const int R = BM + (C2D ? 2 * p.row2d + 2 : (Kr - 1) * dil);
    const int nstep1 = G == 4 ? nchunk >> 2 : (G == 2 ? nchunk >> 1 : nchunk);     // GEMM-1 steps
    const uint32_t a_plane = (uint32_t)G * T1::KG * Rpad * 16, a_bytes = a_plane * T1::planes;
    uint8_t* abuf = smem + kSmemHdr;
    float4* master = reinterpret_cast<float4*>(abuf + 2 * (size_t)a_bytes);
    const uint32_t m_bytes = master_bytes(PROMO, nchunk, p.promote_every, NI);
    uint8_t* wbuf = abuf + 2 * (size_t)a_bytes + m_bytes;
    // a promoted unit's GEMM-2 operand (4 C BM bytes, the master's size at N = C) takes the master's place: the master is
    // dead after GEMM 1's last promotion
    uint8_t* a2buf = m_bytes ? reinterpret_cast<uint8_t*>(master) : wbuf + (size_t)S * p.b_slot;
    const uint32_t w_unit1 = (uint32_t)Kr * T1::planes * T1::KG * N * 16;
    const uint32_t w_unit2 = FUSED ? (uint32_t)prec_planes(P2) * prec_kg(P2) * N * 16 : 0;
    const int units = nstep1 + (FUSED ? p.nchunk2 : 0);

    if (tid == 0) {
        for (int i = 0; i < S; ++i) mbar_init(&full[i], 1);
        fence_mbar_init();
    }
    __syncthreads();
    auto issue_w = [&](int u) {
        uint64_t* bar = &full[u % S];
        uint8_t* dst = wbuf + (size_t)(u % S) * p.b_slot;
        const uint8_t* src;
        uint32_t bytes;
        if (u < nstep1) {
            src = reinterpret_cast<const uint8_t*>(p.wblob) + ((size_t)ntile * nchunk + (size_t)u * G) * w_unit1;
            bytes = G * w_unit1;
        } else { src = reinterpret_cast<const uint8_t*>(p.wblob2) + (size_t)(u - nstep1) * w_unit2; bytes = w_unit2; }
        mbar_arrive_expect_tx(bar, bytes);
        bulk_g2s(dst, src, bytes, bar);
    };
    if (tid == 0)
        for (int u = 0; u < S - 1 && u < units; ++u) issue_w(u);

    const PadMap pm = PadMap::lane(p.lane_len, b, p.Tin, p.pad_left_s, p.pad_right_s, p.reflect);
    const float* __restrict__ xb = p.x + (size_t)b * p.x_bstride;
    auto produce = [&](int s) {              // the operand of GEMM-1 step s: chunks s*G .. s*G + G - 1
        uint8_t* ahi = abuf + (size_t)(s & 1) * a_bytes;
        auto run = [&](auto grouped) {
            constexpr bool GR = decltype(grouped)::value;
            const int c = GR ? s * G : s;
            if constexpr (P1 == P_TF32) produce_chunk<kThreads, GR, false>(p, pm, xb, c, G, t0, R, Rpad, ahi, ahi + a_plane, tid);
            else if constexpr (P1 == P_BF16) produce_chunk<kThreads, GR, true>(p, pm, xb, c, G, t0, R, Rpad, ahi, ahi + a_plane, tid);
            else if constexpr (P1 == P_F16S) produce_chunk<kThreads, GR, true, 4, false, false, true>(p, pm, xb, c, G, t0, R, Rpad, ahi, ahi, tid);
            else produce_chunk<kThreads, GR, false, 4, false, true>(p, pm, xb, c, G, t0, R, Rpad, ahi, ahi + a_plane, tid);
        };
        if constexpr (GROUPABLE) {
            if (G > 1) run(std::true_type());
            else run(std::false_type());
        } else {
            run(std::false_type());
        }
        fence_proxy_async();    // make the generic-proxy stores visible to the tensor core
    };
    produce(0);

    float acc[NI / 2];                   // promoted: the current window (f16x2: its hi*hi products)
    float crs[F16X2 ? NI / 2 : 1];       // f16x2: the window's 2^11-scaled cross terms
    zero_acc<NI>(acc);
    if constexpr (F16X2) zero_acc<NI>(crs);
    const uint32_t a_lbo = (uint32_t)Rpad * 16, b_lbo = (uint32_t)N * 16;
    const uint32_t abase = smem_u32(abuf), wbase = smem_u32(wbuf), a2base = smem_u32(a2buf);
    const int BM2 = BM;

    // master += window (f16x2: hi*hi + cross * 2^-11), in fp32.  The first window adds to zero without reading the master;
    // the last leaves the total in acc for the epilogue without writing it.  Thread-private slots need no barrier.
    auto promote = [&](bool first, bool last) {
        if constexpr (PROMO) {
#pragma unroll
            for (int q = 0; q < NI / 8; ++q) {
                float w[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int i = 4 * q + e;
                    if constexpr (F16X2) { w[e] = acc[i] + crs[i] * kLoUnscale; crs[i] = 0.f; }
                    else w[e] = acc[i];
                }
                float4 m = first ? make_float4(0.f, 0.f, 0.f, 0.f) : master[q * kThreads + tid];
                m.x += w[0]; m.y += w[1]; m.z += w[2]; m.w += w[3];
                if (!last) master[q * kThreads + tid] = m;
                acc[4 * q + 0] = last ? m.x : 0.f;
                acc[4 * q + 1] = last ? m.y : 0.f;
                acc[4 * q + 2] = last ? m.z : 0.f;
                acc[4 * q + 3] = last ? m.w : 0.f;
            }
        }
    };

#pragma unroll 1
    for (int u = 0; u < units; ++u) {
        __syncthreads();                     // operand u ready in every thread's view; the slot refilled below is idle
        if (tid == 0 && u + S - 1 < units) issue_w(u + S - 1);
        mbar_wait(&full[u % S], (uint32_t)(u / S) & 1u);
        const uint32_t wslot = wbase + (uint32_t)(u % S) * p.b_slot;
        wg_fence();
        if (u < nstep1) {
            const uint32_t a0 = abase + (uint32_t)(u & 1) * a_bytes + (uint32_t)tl.row0 * 16;
            const uint32_t b0 = wslot + (uint32_t)tl.col0 * 16;
            auto mma_tap = [&](uint32_t ahi, uint32_t bhi) {    // one tap of one chunk: every split pass
                const uint32_t alo = ahi + a_plane, blo = bhi + T1::KG * b_lbo;
                if constexpr (TT) {         // D[channel][time]: weights are the A operand, activations the B operand
                    mma_pass<P1, NI>(acc, bhi, b_lbo, ahi, a_lbo);
                    mma_pass<P1, NI>(crs, bhi, b_lbo, alo, a_lbo);
                    mma_pass<P1, NI>(crs, blo, b_lbo, ahi, a_lbo);
                } else if constexpr (P1 == P_F16S) {
                    mma_pass<P1, NI>(acc, ahi, a_lbo, bhi, b_lbo);
                } else if constexpr (F16X2) {
                    mma_pass<P1, NI>(acc, ahi, a_lbo, bhi, b_lbo);
                    mma_pass<P1, NI>(crs, ahi, a_lbo, blo, b_lbo);
                    mma_pass<P1, NI>(crs, alo, a_lbo, bhi, b_lbo);
                } else {
                    mma_pass<P1, NI>(acc, ahi, a_lbo, bhi, b_lbo);
                    mma_pass<P1, NI>(acc, ahi, a_lbo, blo, b_lbo);
                    mma_pass<P1, NI>(acc, alo, a_lbo, bhi, b_lbo);
                }
            };
            // One MMA loop per instantiation: a second loop next to it makes ptxas fence every wgmma on its own.
            if constexpr (GROUPABLE) {
                // (chunk, tap) pairs in chunk-major order, so each output element sums its products as one-chunk steps do
                uint32_t ac = a0, bc = b0, ahi = a0, bhi = b0;     // the chunk's and the tap's operand starts
#pragma unroll 1
                for (int i = 0, tap = 0; i < G * Kr; ++i) {
                    mma_tap(ahi, bhi);
                    if (++tap < Kr) { ahi += (uint32_t)dil * 16; bhi += T1::planes * T1::KG * b_lbo; }
                    else { tap = 0; ac += T1::KG * a_lbo; bc += w_unit1; ahi = ac; bhi = bc; }
                }
            } else {
#pragma unroll 1
                for (int tap = 0; tap < Kr; ++tap)
                    mma_tap(a0 + (uint32_t)(C2D ? (tap / 3) * p.row2d + tap % 3 : tap * dil) * 16,
                            b0 + (uint32_t)tap * T1::planes * T1::KG * b_lbo);
            }
            wg_commit();
            if (u + 1 < nstep1) produce(u + 1);         // overlaps the MMAs in flight
            wg_wait_all();
            const int done = (u + 1) * G;               // chunks summed so far
            if (PROMO && (done % p.promote_every == 0 || done == nchunk)) promote(done <= p.promote_every, done == nchunk);
            if constexpr (FUSED) {
                if (u + 1 == nstep1) {
                    // GEMM-2 operand snake2(D1 + b7), split, K-major [plane][k-piece][BM rows][16 B]
                    constexpr int KG2 = prec_kg(P2 < 0 ? 0 : P2);
                    const uint32_t a2_plane = (uint32_t)(p.nchunk2 * KG2) * BM2 * 16;
                    if (m_bytes) __syncthreads();     // every thread has read its master slots before any operand store
                    for_each_pair<NI, 32>(tl, acc, [&](int row, int col, float v0, float v1) {
                        const float2 bi = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                        const float2 al = __ldg(reinterpret_cast<const float2*>(p.out_alpha + col));
                        const float2 ia = __ldg(reinterpret_cast<const float2*>(p.out_inv_alpha + col));
                        v0 = act_out<DEC>(ACT_SNAKE, v0 + bi.x, al.x, ia.x);
                        v1 = act_out<DEC>(ACT_SNAKE, v1 + bi.y, al.y, ia.y);
                        if constexpr (P2 == P_BF16) {
                            __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);
                            float2 hf = __bfloat1622float2(h);
                            __nv_bfloat162 l = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
                            const uint32_t off = ((uint32_t)(col >> 3) * BM2 + row) * 16 + (col & 7) * 2;
                            *reinterpret_cast<__nv_bfloat162*>(a2buf + off) = h;
                            *reinterpret_cast<__nv_bfloat162*>(a2buf + a2_plane + off) = l;
                        } else if constexpr (P2 == P_F16X2) {     // split_store_f16's split, in the bf16 layout
                            const __half2 h = __floats2half2_rn(v0, v1);
                            const float2 hf = __half22float2(h);
                            const __half2 l = __floats2half2_rn((v0 - hf.x) * kLoScale, (v1 - hf.y) * kLoScale);
                            const uint32_t off = ((uint32_t)(col >> 3) * BM2 + row) * 16 + (col & 7) * 2;
                            *reinterpret_cast<__half2*>(a2buf + off) = h;
                            *reinterpret_cast<__half2*>(a2buf + a2_plane + off) = l;
                        } else {
                            const float h0 = to_tf32(v0), h1 = to_tf32(v1);
                            const uint32_t off = ((uint32_t)(col >> 2) * BM2 + row) * 16 + (col & 3) * 4;
                            *reinterpret_cast<float2*>(a2buf + off) = make_float2(h0, h1);
                            *reinterpret_cast<float2*>(a2buf + a2_plane + off) = make_float2(to_tf32(v0 - h0), to_tf32(v1 - h1));
                        }
                    });
                    fence_proxy_async();
                    zero_acc<NI>(acc);
                }
            }
        } else if constexpr (FUSED) {
            constexpr int P2x = P2 < 0 ? 0 : P2;
            constexpr int KG2 = prec_kg(P2x);
            const int c2 = u - nstep1;
            const uint32_t a2_plane = (uint32_t)(p.nchunk2 * KG2) * BM2 * 16, a2_lbo = (uint32_t)BM2 * 16;
            const uint32_t ahi = a2base + ((uint32_t)(c2 * KG2) * BM2 + tl.row0) * 16, alo = ahi + a2_plane;
            const uint32_t bhi = wslot + (uint32_t)tl.col0 * 16, blo = bhi + KG2 * b_lbo;
            if constexpr (P2x == P_F16X2) {      // the unfused 1x1's passes and order; its K loop is one promotion window
                mma_pass<P2x, NI>(acc, ahi, a2_lbo, bhi, b_lbo);
                mma_pass<P2x, NI>(crs, ahi, a2_lbo, blo, b_lbo);
                mma_pass<P2x, NI>(crs, alo, a2_lbo, bhi, b_lbo);
            } else {
                mma_pass<P2x, NI>(acc, ahi, a2_lbo, bhi, b_lbo);
                mma_pass<P2x, NI>(acc, ahi, a2_lbo, blo, b_lbo);
                mma_pass<P2x, NI>(acc, alo, a2_lbo, bhi, b_lbo);
            }
            wg_commit();
            wg_wait_all();
            if (PROMO && c2 + 1 == p.nchunk2) promote(true, true);
        }
    }

    // ================= epilogue =================
    const float* __restrict__ bias = FUSED ? p.bias2 : p.bias;
    const int act = FUSED ? ACT_NONE : p.out_act;
    float* __restrict__ yb = p.y + (size_t)b * p.y_bstride + (size_t)ntile * N;
    const float* __restrict__ rb = p.res ? p.res + (size_t)b * p.y_bstride + (size_t)ntile * N : nullptr;
    const float* al_p = act == ACT_SNAKE ? p.out_alpha + (size_t)ntile * N : nullptr;
    const float* ia_p = act == ACT_SNAKE ? p.out_inv_alpha + (size_t)ntile * N : nullptr;
    const float* bi_p = bias ? bias + (size_t)ntile * N : nullptr;
    if constexpr (TT) {
        // fragment row = output channel, column = time step
        for_each_pair<NI>(tl, acc, [&](int r, int c, float v0, float v1) {
            if (r - tl.row0 >= NW) return;           // A-operand rows past this warpgroup's channels
            const int co = tl.col0 + (r - tl.row0), tf = tl.row0 + (c - tl.col0);
            const float bi = bi_p ? __ldg(bi_p + co) : 0.f;
            const float al = act == ACT_SNAKE ? __ldg(al_p + co) : 0.f, ia = act == ACT_SNAKE ? __ldg(ia_p + co) : 0.f;
            const float v[2] = {v0, v1};
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int t = t0 + tf + e;
                if (t >= p.Tout) continue;
                float o = act_out<DEC>(act, v[e] + bi, al, ia);
                if (rb) o += rb[(size_t)t * p.ldy + co];
                yb[(size_t)t * p.ldy + co] = o;
            }
        });
        return;
    }
    for_each_pair<NI>(tl, acc, [&](int row, int col, float v0, float v1) {
        const int t = t0 + row;
        if (t >= p.Tout) return;
        if constexpr (C2D) {
            const float2 bi = __ldg(reinterpret_cast<const float2*>(bi_p + col));
            v0 += bi.x; v1 += bi.y;
            if (act == ACT_LRELU) { v0 = v0 >= 0.f ? v0 : 0.01f * v0; v1 = v1 >= 0.f ? v1 : 0.01f * v1; }
            if (rb) { const float2 r = *reinterpret_cast<const float2*>(rb + (size_t)t * p.ldy + col); v0 += r.x; v1 += r.y; }
            const int f = t % p.row2d;
            if (f == 0 || f == p.row2d - 1) { v0 = 0.f; v1 = 0.f; }
            *reinterpret_cast<float2*>(yb + (size_t)t * p.ldy + col) = make_float2(v0, v1);
            return;
        }
        if (bi_p) { const float2 bi = __ldg(reinterpret_cast<const float2*>(bi_p + col)); v0 += bi.x; v1 += bi.y; }
        if (act == ACT_SNAKE) {
            const float2 al = __ldg(reinterpret_cast<const float2*>(al_p + col));
            const float2 ia = __ldg(reinterpret_cast<const float2*>(ia_p + col));
            v0 = act_out<DEC>(ACT_SNAKE, v0, al.x, ia.x);
            v1 = act_out<DEC>(ACT_SNAKE, v1, al.y, ia.y);
        } else if (act != ACT_NONE) {
            v0 = act_out<DEC>(act, v0, 0.f, 0.f);
            v1 = act_out<DEC>(act, v1, 0.f, 0.f);
        }
        if (rb) { const float2 r = *reinterpret_cast<const float2*>(rb + (size_t)t * p.ldy + col); v0 += r.x; v1 += r.y; }
        *reinterpret_cast<float2*>(yb + (size_t)t * p.ldy + col) = make_float2(v0, v1);
    });
}

template <int P1, int P2, bool PROMO, int NI, int MINB = 1, bool TT = false>
__global__ void __launch_bounds__(kThreads, groupable<P1, P2, TT>() && NI <= 128 ? 2 : MINB) conv_tc_kernel(TcConvParams p) {
    conv_tc_body<P1, P2, PROMO, NI, MINB, TT, false>(p);
}

// 3x3 Conv2d (JDCNet, jdc.cu) in the promoted fp16 hi + scaled-lo class, two CTAs per SM where the plan fits
template <int NI>
__global__ void __launch_bounds__(kThreads, 2) conv2d_tc_kernel(TcConvParams p) {
    conv_tc_body<P_F16X2, P_NONE, true, NI, 2, false, true>(p);
}

}  // namespace

// ---- host side ---------------------------------------------------------------------------------
namespace {
constexpr size_t kSmemCap = 227 * 1024;        // dynamic shared memory per block (sm_90)
constexpr size_t kSmemCap2 = 113 * 1024;       // per block with two resident blocks (228 KB per SM, 1 KB reserved each)
int plan_prec(const TcConvParams& p) {
    return p.g1f16 ? P_F16S : (p.f16x2 ? P_F16X2 : (p.bf16 ? P_BF16 : P_TF32));
}
// Warpgroup width above 128 that the one-pass fp16 class is compiled for (launch_conv_tc): 256 for a plain conv (the
// decoder's C = 768 conv7), 192 for a fused unit (the C = 192 ResidualUnit).  A plain N = 192 k = 7 conv fits two 64-row
// CTAs per SM and keeps them (tc_conv_plan); a fused unit at C = 256 has no room for two weight slots next to its 128-row
// GEMM-2 operand, and the 64-row plan with two slots comes first.
constexpr int f16s_wide_nw(bool fused) { return fused ? 192 : 256; }
}  // namespace

bool tc_conv_plan(TcConvParams& p) {
    // p.Cin, p.vf, p.Kr, p.dil, p.Cout, p.promoted (+ bf16 / g1f16 / f16x2 / fused / tt / occ2_maxn) must be set; fills N,
    // MT, nchunk, Rpad, stagesB, b_slot, smem_bytes, promote_every, occ2, group
    if ((p.Cin % 4) != 0 || ((p.Cin * p.vf) % kChunk) != 0 || (p.Cout % 16) != 0) return false;
    if (p.bf16 && p.promoted) return false;
    if (p.f16x2 && !p.promoted) return false;
    if (p.g1f16 && !p.bf16) return false;
    if (p.tt && !p.f16x2) return false;
    if (p.row2d && (p.Kr != 9 || p.vf != 1 || !p.f16x2 || p.tt || p.fused || p.row2d < 3)) return false;
    if (p.fused && ((p.promoted && (!p.f16x2 || p.tt)) || p.Cin != p.Cout || p.vf != 1 || p.Cout > 256)) return false;
    const int P1 = plan_prec(p), P2 = p.fused ? (p.f16x2 ? P_F16X2 : (p.bf16 ? P_BF16 : P_TF32)) : P_NONE;
    p.nchunk = p.Cin * p.vf / kChunk;
    p.nchunk2 = p.fused ? p.Cout / kChunk : 0;
    p.promote_every = p.promoted ? (p.f16x2 ? (48 / p.Kr < 1 ? 1 : 48 / p.Kr) : (8 / p.Kr < 1 ? 1 : 8 / p.Kr)) : 1;
    // A promoted unit's GEMM 2 (the 1x1) promotes once, at its end, as the unfused 1x1 does: one window of <= 48 chunks.
    if (p.fused && p.promoted && p.nchunk2 > 48) return false;
    const int nw_max = p.promoted ? 64 : 128;      // accumulator registers per thread: NW / 2 (x 3 when promoted)
    // N depends on the layer's shape and split class only (never on dil, Tout, tt or occ2_maxn): the weight blob is laid
    // out for it once (tc_pack_blob) and every later plan of the layer must find the same N.  It is the widest tile whose
    // weight slot and fused GEMM-2 operand leave kAReserve bytes for the activation buffers; a fused unit needs N = C.
    constexpr size_t kAReserve = 40 * 1024;
    int N = 0;
    for (int cand = p.fused ? p.Cout : 256; cand >= 16 && N == 0; cand -= 16) {
        const bool rows_split = cand <= nw_max, cols_split = (cand / 2) % 16 == 0 && cand / 2 <= nw_max;
        if (p.Cout % cand || !(rows_split || cols_split)) continue;
        size_t slot = (size_t)p.Kr * prec_planes(P1) * prec_kg(P1) * cand * 16, a2 = 0;
        if (P2 != P_NONE) a2 = (size_t)prec_planes(P2) * p.nchunk2 * prec_kg(P2) * 64 * 16;
        if (kSmemHdr + kAReserve + slot + a2 <= kSmemCap) N = cand;
        else if (p.fused) return false;
    }
    if (N == 0 || (p.fused && p.promoted && N != p.Cout)) return false;
    // Two resident CTAs per SM: one CTA's operand production, barriers, promotions and epilogue overlap the other's MMAs;
    // each gets half the shared memory and <= 128 registers per thread.  Always tried for the promoted class, which loses
    // no MMA width to it (NW <= 64 either way); for the others only for tiles of N <= occ2_maxn, which must halve NW.
    // The one-pass fp16 class (g1f16) does ONE MMA per streamed weight element, against three in the split classes, so
    // it needs three times the weight bytes per MMA clock.  Where its 64-row tile runs one CTA per SM anyway (more than
    // half the shared memory), it takes the N of f16s_wide_nw as 128 rows with each warpgroup over all N channels (NW = N,
    // m64n192 / m64n256 accumulators of 96 / 128 registers): both warpgroups then read every weight chunk, which halves
    // the weight bytes per MMA, and the per-chunk barrier, weight wait and halo rows are amortized over twice the rows.
    // A 64-row tile that fits two CTAs per SM (its kernel has <= 128 registers at NW <= 128) keeps them: the other CTA's
    // MMAs then cover those same costs (the C = 384 conv7 at the bench workload: 2.2 ms in two 64-row CTAs per SM, 3.1 ms
    // in one 128-row CTA; H100 80GB HBM3, 700 W, 1980 MHz max SM clock).  N itself is what the loop above found, so the
    // weight blob does not change.
    struct Layout { int Rpad; size_t slot, total; };
    auto layout = [&](int S, int MT, int G) {
        const int NW = MT == 2 ? N : N / 2, BM = 64 * MT;
        Layout l;
        // Row pitch: one store phase of the producer (8 threads of 16-byte TF32 pieces, 16 threads of 8-byte 16-bit pieces)
        // covers v rows x 8/v pitch-apart columns of 16 bytes, conflict-free when Rpad % 8 == v: v = 1 for TF32 at G > 1,
        // 4/G in the 16-bit classes at G > 1.  G = 1 keeps Rpad % 8 == 2, right for TF32 (v = 2) and a 2-way conflict
        // in the 16-bit classes (v = 4), as the one-chunk plans have always been laid out.
        const int v = G == 1 ? 2 : (P1 == P_TF32 ? 1 : 4 / G);
        l.Rpad = BM + (p.row2d ? 2 * p.row2d + 2 : (p.Kr - 1) * p.dil);
        while (l.Rpad % 8 != v) ++l.Rpad;
        const size_t a_bytes = (size_t)G * prec_planes(P1) * prec_kg(P1) * l.Rpad * 16;
        l.slot = (size_t)G * p.Kr * prec_planes(P1) * prec_kg(P1) * N * 16;
        size_t a2 = 0;
        if (P2 != P_NONE) {
            const size_t slot2 = (size_t)prec_planes(P2) * prec_kg(P2) * N * 16;
            if (slot2 > l.slot) l.slot = slot2;
            a2 = (size_t)prec_planes(P2) * p.nchunk2 * prec_kg(P2) * BM * 16;
        }
        // transposed: a warpgroup's A operand is always 64 channel rows; rows past its NW read (and discard) whatever
        // follows the weight slot, so the buffer ends with 64 rows of slack
        const size_t master = master_bytes(p.promoted, p.nchunk, p.promote_every, p.tt ? 64 : NW);
        if (master) a2 = 0;     // a promoted unit's GEMM-2 operand aliases the master: both are 4 C BM bytes at N = C
        l.total = kSmemHdr + 2 * a_bytes + master + S * l.slot + a2 + (p.tt ? 64 * 16 : 0);
        return l;
    };
    // Chunks per K-loop step G: every step pays a barrier, a weight wait, a global-load round trip for the next operand
    // and a tensor-pipe drain, which a k = 7 conv's 7 taps of MMAs hide and a layer of 1-3 taps does not.  Such a layer
    // streams G consecutive chunks per step (their weights are contiguous in the blob) into G-times larger operand and
    // weight slots, as long as the plan keeps its residency: a plan within half the shared memory (two CTAs per SM, the
    // register budget of every <= 128-column instantiation allows it) stays within it.  G divides the promotion window,
    // so windows close at the same chunks; the transposed formulation keeps one chunk per step.
    auto group = [&](int S, int MT, size_t cap) {
        if (p.Kr > 3 || p.tt || p.fused || p.g1f16) return 1;     // the instantiations without the grouped loop
        for (int G = 4; G > 1; G /= 2)
            if (G <= p.max_group && p.nchunk % G == 0 && (!p.promoted || p.promote_every % G == 0) && layout(S, MT, G).total <= cap) return G;
        return 1;
    };
    // A promoted unit is planned for two CTAs per SM or not at all: at one CTA per SM it would give back more than fusing
    // saves (two CTAs per SM gave the promoted k = 7 convs 18-43 %).  Its kernel is compiled for NW = 64 only: C = 64 as
    // 128 rows, C = 128 as 64 rows, the tiles of the unit's two unfused convs.
    const bool unit2 = p.fused && p.promoted;
    const bool want2 = p.promoted ? !p.tt : (p.occ2_maxn > 0 && N <= p.occ2_maxn);
    for (int two = want2 ? 1 : 0; two >= (unit2 ? 1 : 0); --two) {
        const size_t cap = two ? kSmemCap2 : kSmemCap;
        const int nwl = two ? 64 : nw_max;
        for (int S = 2; S >= 1; --S)
            for (int MT = 2; MT >= 1; --MT) {
                const int NW = MT == 2 ? N : N / 2;
                const bool wide = !two && P1 == P_F16S && NW == f16s_wide_nw(p.fused);
                if ((NW > nwl && !wide) || NW % 16 || (unit2 && NW != 64)) continue;
                if (wide && layout(2, 1, 1).total <= kSmemCap2) continue;
                const Layout l1 = layout(S, MT, 1);
                if (l1.total > cap) continue;
                const int G = group(S, MT, l1.total <= kSmemCap2 ? kSmemCap2 : cap);
                const Layout l = layout(S, MT, G);
                p.N = N; p.MT = MT; p.Rpad = l.Rpad; p.R2pad = 64 * MT; p.stagesB = S; p.b_slot = (int)l.slot;
                p.group = G;
                p.smem_bytes = l.total;
                p.occ2 = two;
                return true;
            }
    }
    return false;
}

size_t tc_blob_floats(const TcConvParams& p) {
    if (p.g1f16) return (size_t)(p.Cout / p.N) * p.nchunk * p.Kr * 2 * p.N * 4;     // hi plane only
    return (size_t)(p.Cout / p.N) * p.nchunk * p.Kr * 2 * ((p.bf16 || p.f16x2) ? 2 : 4) * p.N * 4;
}

static inline uint16_t bf16_rn_host(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    u += 0x7FFFu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}

// wp: packed generic weights [Kr * vf*Cin][ldw] (conv_simt layout).  blob: see file header.
void tc_pack_blob(const TcConvParams& p, const float* wp, int ldw, float* blob) {
    const int Cw = p.Cin * p.vf;   // columns per row-tap
    if (p.g1f16) {
        // [ntile][chunk][tap][k8 (2)][N][8 fp16]: rn_f16(w) only
        uint16_t* ob = reinterpret_cast<uint16_t*>(blob);
        size_t o16 = 0;
        for (int nt = 0; nt < p.Cout / p.N; ++nt)
            for (int c = 0; c < p.nchunk; ++c)
                for (int tap = 0; tap < p.Kr; ++tap)
                    for (int k8 = 0; k8 < 2; ++k8)
                        for (int n = 0; n < p.N; ++n)
                            for (int e = 0; e < 8; ++e) {
                                int kk = tap * Cw + c * tc::kChunk + k8 * 8 + e;
                                __half v = __float2half_rn(wp[(size_t)kk * ldw + nt * p.N + n]);
                                uint16_t bits;
                                memcpy(&bits, &v, 2);
                                ob[o16++] = bits;
                            }
        return;
    }
    if (p.f16x2) {
        // [ntile][chunk][tap][hi|lo'][k8 (2)][N][8 fp16], lo' = rn_f16((w - hi) * 2^11)
        uint16_t* ob = reinterpret_cast<uint16_t*>(blob);
        size_t o16 = 0;
        for (int nt = 0; nt < p.Cout / p.N; ++nt)
            for (int c = 0; c < p.nchunk; ++c)
                for (int tap = 0; tap < p.Kr; ++tap)
                    for (int hl = 0; hl < 2; ++hl)
                        for (int k8 = 0; k8 < 2; ++k8)
                            for (int n = 0; n < p.N; ++n)
                                for (int e = 0; e < 8; ++e) {
                                    int kk = tap * Cw + c * tc::kChunk + k8 * 8 + e;
                                    float w = wp[(size_t)kk * ldw + nt * p.N + n];
                                    __half hi = __float2half_rn(w);
                                    __half v = hl == 0 ? hi : __float2half_rn((w - __half2float(hi)) * 2048.0f);
                                    uint16_t bits;
                                    memcpy(&bits, &v, 2);
                                    ob[o16++] = bits;
                                }
        return;
    }
    if (p.bf16) {
        // [ntile][chunk][tap][hi|lo][k8 (2)][N][8 bf16]
        uint16_t* ob = reinterpret_cast<uint16_t*>(blob);
        size_t o16 = 0;
        for (int nt = 0; nt < p.Cout / p.N; ++nt)
            for (int c = 0; c < p.nchunk; ++c)
                for (int tap = 0; tap < p.Kr; ++tap)
                    for (int hl = 0; hl < 2; ++hl)
                        for (int k8 = 0; k8 < 2; ++k8)
                            for (int n = 0; n < p.N; ++n)
                                for (int e = 0; e < 8; ++e) {
                                    int kk = tap * Cw + c * tc::kChunk + k8 * 8 + e;
                                    float w = wp[(size_t)kk * ldw + nt * p.N + n];
                                    uint16_t hi = bf16_rn_host(w);
                                    uint32_t hu = (uint32_t)hi << 16;
                                    float hf;
                                    memcpy(&hf, &hu, 4);
                                    ob[o16++] = hl == 0 ? hi : bf16_rn_host(w - hf);
                                }
        return;
    }
    size_t o = 0;
    for (int nt = 0; nt < p.Cout / p.N; ++nt)
        for (int c = 0; c < p.nchunk; ++c)
            for (int tap = 0; tap < p.Kr; ++tap)
                for (int hl = 0; hl < 2; ++hl)
                    for (int k4 = 0; k4 < 4; ++k4)
                        for (int n = 0; n < p.N; ++n)
                            for (int e = 0; e < 4; ++e) {
                                int kk = tap * Cw + c * tc::kChunk + k4 * 4 + e;
                                float w = wp[(size_t)kk * ldw + nt * p.N + n];
                                // round-to-nearest-even-ish TF32 split (ties away, like cvt.rna)
                                uint32_t u;
                                memcpy(&u, &w, 4);
                                uint32_t hu = (u + 0x1000u) & 0xFFFFE000u;
                                float hi;
                                memcpy(&hi, &hu, 4);
                                float lo = w - hi;
                                uint32_t lu;
                                memcpy(&lu, &lo, 4);
                                lu = (lu + 0x1000u) & 0xFFFFE000u;
                                float lo_r;
                                memcpy(&lo_r, &lu, 4);
                                blob[o++] = hl == 0 ? hi : lo_r;
                            }
}

namespace {
template <int P1, int P2, bool PROMO, int NI, int MINB = 1, bool TT = false, bool C2D = false>
cudaError_t launch_one(const TcConvParams& p, dim3 grid, cudaStream_t st) {
    auto* kern = [] {
        if constexpr (C2D) return conv2d_tc_kernel<NI>;
        else return conv_tc_kernel<P1, P2, PROMO, NI, MINB, TT>;
    }();
    // the > 48 KB dynamic shared-memory opt-in is per device and per kernel
    static bool done[64] = {};
    static std::mutex mu;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (!done[dev]) {
            e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap);
            if (e != cudaSuccess) return e;
            done[dev] = true;
        }
    }
    kern<<<grid, kThreads, p.smem_bytes, st>>>(p);
    return cudaGetLastError();
}
// The kernel's wgmma N is the warpgroup's whole channel width NW, so there is one instantiation per width tc_conv_plan
// can return for the class: 16, 32, ..., 128, or up to 64 when promoted or planned for two CTAs per SM, plus
// f16s_wide_nw in the one-pass fp16 class.  The promoted class (TT aside) has only the MINB = 2
// instantiations, whatever residency its plan allows.
template <int P1, int P2, bool PROMO, int MINB = 1, int NI = (PROMO || MINB == 2 ? 64 : 128), bool C2D = false>
cudaError_t launch_nw(const TcConvParams& p, dim3 grid, cudaStream_t st) {
    const int NW = p.MT == 2 ? p.N : p.N / 2;
    if (NW == NI) return launch_one<P1, P2, PROMO, NI, MINB, false, C2D>(p, grid, st);
    if constexpr (NI > 16) return launch_nw<P1, P2, PROMO, MINB, NI - 16, C2D>(p, grid, st);
    else return cudaErrorInvalidValue;
}
template <int P1, int P2>
cudaError_t launch_occ(const TcConvParams& p, dim3 grid, cudaStream_t st) {
    if (p.occ2) return launch_nw<P1, P2, false, 2>(p, grid, st);
    if constexpr (P1 == P_F16S) {
        constexpr int kWide = f16s_wide_nw(P2 != P_NONE);
        if ((p.MT == 2 ? p.N : p.N / 2) == kWide) return launch_one<P1, P2, false, kWide>(p, grid, st);
    }
    return launch_nw<P1, P2, false, 1>(p, grid, st);
}
}  // namespace

cudaError_t launch_conv_tc(const TcConvParams& p, cudaStream_t st) {
    if (p.Tout <= 0 || p.B <= 0) return cudaSuccess;
    const int BM = 64 * p.MT;
    dim3 grid((p.Tout + BM - 1) / BM, p.Cout / p.N, p.B);
    if (grid.y > 65535 || grid.z > 65535) return cudaErrorInvalidValue;
    const int P1 = plan_prec(p);
    if (p.row2d) {
        if (P1 != P_F16X2 || !p.promoted || p.fused || p.tt || p.Kr != 9) return cudaErrorInvalidValue;
        return launch_nw<P_F16X2, P_NONE, true, 2, 64, true>(p, grid, st);
    }
    if (p.fused) {
        if (P1 == P_F16X2)
            return (p.MT == 2 ? p.N : p.N / 2) == 64 ? launch_one<P_F16X2, P_F16X2, true, 64, 2>(p, grid, st) : cudaErrorInvalidValue;
        if (P1 == P_F16S) return launch_occ<P_F16S, P_BF16>(p, grid, st);
        if (P1 == P_BF16) return launch_occ<P_BF16, P_BF16>(p, grid, st);
        return launch_occ<P_TF32, P_TF32>(p, grid, st);
    }
    if (p.tt) return launch_one<P_F16X2, P_NONE, true, 64, 1, true>(p, grid, st);
    if (p.promoted)
        return P1 == P_F16X2 ? launch_nw<P_F16X2, P_NONE, true, 2>(p, grid, st) : launch_nw<P_TF32, P_NONE, true, 2>(p, grid, st);
    if (P1 == P_F16S) return launch_occ<P_F16S, P_NONE>(p, grid, st);
    if (P1 == P_BF16) return launch_occ<P_BF16, P_NONE>(p, grid, st);
    return launch_occ<P_TF32, P_NONE>(p, grid, st);
}

}  // namespace fac
