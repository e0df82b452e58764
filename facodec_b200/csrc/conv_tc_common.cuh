// mbarrier / bulk-copy / wgmma primitives and the activation-operand producer of the tensor-core conv kernel
// (conv_tc.cu).  Device code only.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "kernels.h"

namespace fac {

namespace tc {

constexpr int kThreads = 256;     // two warpgroups: both produce operands, each issues wgmma for its share of the tile
constexpr int kChunk = 16;        // K elements (channels) per pipeline chunk
constexpr int kSmemHdr = 128;     // mbarriers at the start of dynamic shared memory

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Two flavours of waiting: polled back to back (RELAXED = false), or with a short suspend-time hint (0.4 us) that parks
// the thread in hardware between polls.
template <bool RELAXED>
__device__ __forceinline__ bool mbar_try_wait_t(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    if constexpr (RELAXED) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity), "r"(400u)
            : "memory");
    } else {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
    return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel aborts with an error) instead of hanging the GPU.
template <bool RELAXED = false>
__device__ __forceinline__ void mbar_wait_t(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait_t<RELAXED>(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait_t<RELAXED>(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait_t<false>(bar, parity); }
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) { mbar_wait_t<true>(bar, parity); }
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---- wgmma (sm_90a) ------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes stored as 128 contiguous
// bytes; LBO = byte pitch between core matrices adjacent in K, SBO = byte pitch between 8-row groups.
__device__ __forceinline__ uint64_t gdesc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

enum WgKind { WG_TF32 = 0, WG_BF16 = 1, WG_F16 = 2 };

// D[64 x NI] += A[64 x K] * B[NI x K]^T, both operands K-major in shared memory; K = 16 (f16 / bf16) or 8 (tf32).
// Defined for NI = 16, 32, ..., 256 by FAC_WGMMA_SS below; any other NI fails to compile.
template <int NI, int KIND>
__device__ __forceinline__ void wgmma_ss(float (&d)[NI / 2], uint64_t da, uint64_t db) {
    static_assert(NI < 0, "wgmma_ss: instruction N must be a multiple of 16 in [16, 256]");
}

// The m64nNI accumulator is NI/2 registers per thread, listed in groups of 8: FAC_Sg is the asm operand list
// "%0, ..., %(8g-1)" and FAC_Cg the matching "+f" constraints on d[0 .. 8g-1].
#define FAC_S1 "%0, %1, %2, %3, %4, %5, %6, %7"
#define FAC_S2 FAC_S1 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define FAC_S3 FAC_S2 ", %16, %17, %18, %19, %20, %21, %22, %23"
#define FAC_S4 FAC_S3 ", %24, %25, %26, %27, %28, %29, %30, %31"
#define FAC_S5 FAC_S4 ", %32, %33, %34, %35, %36, %37, %38, %39"
#define FAC_S6 FAC_S5 ", %40, %41, %42, %43, %44, %45, %46, %47"
#define FAC_S7 FAC_S6 ", %48, %49, %50, %51, %52, %53, %54, %55"
#define FAC_S8 FAC_S7 ", %56, %57, %58, %59, %60, %61, %62, %63"
#define FAC_S9 FAC_S8 ", %64, %65, %66, %67, %68, %69, %70, %71"
#define FAC_S10 FAC_S9 ", %72, %73, %74, %75, %76, %77, %78, %79"
#define FAC_S11 FAC_S10 ", %80, %81, %82, %83, %84, %85, %86, %87"
#define FAC_S12 FAC_S11 ", %88, %89, %90, %91, %92, %93, %94, %95"
#define FAC_S13 FAC_S12 ", %96, %97, %98, %99, %100, %101, %102, %103"
#define FAC_S14 FAC_S13 ", %104, %105, %106, %107, %108, %109, %110, %111"
#define FAC_S15 FAC_S14 ", %112, %113, %114, %115, %116, %117, %118, %119"
#define FAC_S16 FAC_S15 ", %120, %121, %122, %123, %124, %125, %126, %127"
#define FAC_R8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
    "+f"(d[o + 6]), "+f"(d[o + 7])
#define FAC_C1 FAC_R8(0)
#define FAC_C2 FAC_C1, FAC_R8(8)
#define FAC_C3 FAC_C2, FAC_R8(16)
#define FAC_C4 FAC_C3, FAC_R8(24)
#define FAC_C5 FAC_C4, FAC_R8(32)
#define FAC_C6 FAC_C5, FAC_R8(40)
#define FAC_C7 FAC_C6, FAC_R8(48)
#define FAC_C8 FAC_C7, FAC_R8(56)
#define FAC_C9 FAC_C8, FAC_R8(64)
#define FAC_C10 FAC_C9, FAC_R8(72)
#define FAC_C11 FAC_C10, FAC_R8(80)
#define FAC_C12 FAC_C11, FAC_R8(88)
#define FAC_C13 FAC_C12, FAC_R8(96)
#define FAC_C14 FAC_C13, FAC_R8(104)
#define FAC_C15 FAC_C14, FAC_R8(112)
#define FAC_C16 FAC_C15, FAC_R8(120)
// One specialization per kind for N = 16 * G; the descriptors are operands %(8G) and %(8G + 1), spelled out as DESC.
#define FAC_WGMMA_KIND(N, G, DESC, KIND, SHAPE, TAIL)                                                                   \
    template <>                                                                                                      \
    __device__ __forceinline__ void wgmma_ss<N, KIND>(float (&d)[N / 2], uint64_t da, uint64_t db) {                  \
        asm volatile("wgmma.mma_async.sync.aligned.m64n" #N SHAPE " {" FAC_S##G "}, " DESC ", " TAIL ";"              \
                     : FAC_C##G : "l"(da), "l"(db));                                                                 \
    }
#define FAC_WGMMA_SS(N, G, DESC)                                                                                     \
    FAC_WGMMA_KIND(N, G, DESC, WG_TF32, "k8.f32.tf32.tf32", "1, 1, 1")                                                \
    FAC_WGMMA_KIND(N, G, DESC, WG_BF16, "k16.f32.bf16.bf16", "1, 1, 1, 0, 0")                                         \
    FAC_WGMMA_KIND(N, G, DESC, WG_F16, "k16.f32.f16.f16", "1, 1, 1, 0, 0")
FAC_WGMMA_SS(16, 1, "%8, %9")
FAC_WGMMA_SS(32, 2, "%16, %17")
FAC_WGMMA_SS(48, 3, "%24, %25")
FAC_WGMMA_SS(64, 4, "%32, %33")
FAC_WGMMA_SS(80, 5, "%40, %41")
FAC_WGMMA_SS(96, 6, "%48, %49")
FAC_WGMMA_SS(112, 7, "%56, %57")
FAC_WGMMA_SS(128, 8, "%64, %65")
FAC_WGMMA_SS(144, 9, "%72, %73")
FAC_WGMMA_SS(160, 10, "%80, %81")
FAC_WGMMA_SS(176, 11, "%88, %89")
FAC_WGMMA_SS(192, 12, "%96, %97")
FAC_WGMMA_SS(208, 13, "%104, %105")
FAC_WGMMA_SS(224, 14, "%112, %113")
FAC_WGMMA_SS(240, 15, "%120, %121")
FAC_WGMMA_SS(256, 16, "%128, %129")
#undef FAC_WGMMA_SS
#undef FAC_WGMMA_KIND
#undef FAC_R8
#undef FAC_S1
#undef FAC_S2
#undef FAC_S3
#undef FAC_S4
#undef FAC_S5
#undef FAC_S6
#undef FAC_S7
#undef FAC_S8
#undef FAC_S9
#undef FAC_S10
#undef FAC_S11
#undef FAC_S12
#undef FAC_S13
#undef FAC_S14
#undef FAC_S15
#undef FAC_S16
#undef FAC_C1
#undef FAC_C2
#undef FAC_C3
#undef FAC_C4
#undef FAC_C5
#undef FAC_C6
#undef FAC_C7
#undef FAC_C8
#undef FAC_C9
#undef FAC_C10
#undef FAC_C11
#undef FAC_C12
#undef FAC_C13
#undef FAC_C14
#undef FAC_C15
#undef FAC_C16

__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}


// hi/lo split of 4 consecutive channels of one row + store into the K-major operand buffers.
//   TF32 (BF16 = false): hi = rna_tf32(x), lo = rna_tf32(x - hi); 16-byte piece pc of 4 per 16-channel chunk.
//   BF16 (BF16 = true) : hi = rn_bf16(x), lo = rn_bf16(x - hi) (16 mantissa bits in total: used downstream of the
//   VQ only); 8 bytes = half of 16-byte k-group pc/2 (a k-group is 8 bf16 channels).
template <bool BF16>
__device__ __forceinline__ void split_store(float4 x4, int pc, int row, int Rpad, uint8_t* ahi, uint8_t* alo) {
    if constexpr (!BF16) {
        float4 hi, lo;
        hi.x = to_tf32(x4.x); lo.x = to_tf32(x4.x - hi.x);
        hi.y = to_tf32(x4.y); lo.y = to_tf32(x4.y - hi.y);
        hi.z = to_tf32(x4.z); lo.z = to_tf32(x4.z - hi.z);
        hi.w = to_tf32(x4.w); lo.w = to_tf32(x4.w - hi.w);
        const size_t off = ((size_t)pc * Rpad + row) * 16;
        *reinterpret_cast<float4*>(ahi + off) = hi;
        *reinterpret_cast<float4*>(alo + off) = lo;
    } else {
        __nv_bfloat162 h01 = __floats2bfloat162_rn(x4.x, x4.y), h23 = __floats2bfloat162_rn(x4.z, x4.w);
        float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
        __nv_bfloat162 l01 = __floats2bfloat162_rn(x4.x - f01.x, x4.y - f01.y);
        __nv_bfloat162 l23 = __floats2bfloat162_rn(x4.z - f23.x, x4.w - f23.y);
        const size_t off = ((size_t)(pc >> 1) * Rpad + row) * 16 + (size_t)(pc & 1) * 8;
        uint2 hv, lv;
        hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
        lv.x = *reinterpret_cast<uint32_t*>(&l01); lv.y = *reinterpret_cast<uint32_t*>(&l23);
        *reinterpret_cast<uint2*>(ahi + off) = hv;
        *reinterpret_cast<uint2*>(alo + off) = lv;
    }
}

// fp16 hi + SCALED lo split (conv_tcp_kernel<true>): hi = rn_f16(x), lo' = rn_f16((x - hi) * 2^11).  hi + lo' * 2^-11
// carries 22 mantissa bits like the TF32 pair, but both halves are 16-bit operands of a full-rate kind::f16 MMA; the
// scaling keeps lo' in fp16's normal range (|lo'| <= |x|), and the cross terms are accumulated apart and scaled back
// by 2^-11 at promotion.  Same 8-byte-per-4-channels layout as the bf16 split.
constexpr float kLoScale = 2048.0f, kLoUnscale = 1.0f / 2048.0f;
__device__ __forceinline__ void split_store_f16(float4 x4, int pc, int row, int Rpad, uint8_t* ahi, uint8_t* alo) {
    __half2 h01 = __floats2half2_rn(x4.x, x4.y), h23 = __floats2half2_rn(x4.z, x4.w);
    float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    __half2 l01 = __floats2half2_rn((x4.x - f01.x) * kLoScale, (x4.y - f01.y) * kLoScale);
    __half2 l23 = __floats2half2_rn((x4.z - f23.x) * kLoScale, (x4.w - f23.y) * kLoScale);
    const size_t off = ((size_t)(pc >> 1) * Rpad + row) * 16 + (size_t)(pc & 1) * 8;
    uint2 hv, lv;
    hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
    lv.x = *reinterpret_cast<uint32_t*>(&l01); lv.y = *reinterpret_cast<uint32_t*>(&l23);
    *reinterpret_cast<uint2*>(ahi + off) = hv;
    *reinterpret_cast<uint2*>(alo + off) = lv;
}

// ONE fp16 value per channel (conv_tc_kernel's g1f16 class): hi = rn_f16(x) only, same 8-byte-per-4-channels layout.
__device__ __forceinline__ void store_f16_single(float4 x4, int pc, int row, int Rpad, uint8_t* ahi) {
    __half2 h01 = __floats2half2_rn(x4.x, x4.y), h23 = __floats2half2_rn(x4.z, x4.w);
    const size_t off = ((size_t)(pc >> 1) * Rpad + row) * 16 + (size_t)(pc & 1) * 8;
    uint2 hv;
    hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
    *reinterpret_cast<uint2*>(ahi + off) = hv;
}

// ---- activation producer ----------------------------------------------------------------------
// Chunks c .. c + G - 1 of the operand (GROUPED: G = 2 or 4; else the one chunk c): 4G 16-byte pieces (4 input channels
// each) per row.  Thread `ptid` of NT producer threads owns piece pc = ptid % 4G of rows ptid/4G, ptid/4G + NT/4G, ...:
// channel offset, Snake parameters and the smem column are per-thread constants for the whole call; only the row varies.
// Piece pc lands in k-piece pc (TF32) or pc/2 (16-bit classes) of the buffer, so chunk c + s starts at k-piece s * KG.
template <int NT, bool GROUPED, bool BF16, int BATCH = 4, bool INL = false, bool F16 = false, bool SINGLE = false>
__device__ __forceinline__ void produce_chunk(const TcConvParams& p, const PadMap& pm, const float* __restrict__ xb,
                                              int c, int G, int t0, int R, int Rpad, uint8_t* ahi, uint8_t* alo, int ptid) {
    const int lp = GROUPED ? (G == 4 ? 4 : 3) : 2;           // log2 of the pieces per row
    const int pc = ptid & ((1 << lp) - 1);
    const int j = c * kChunk + pc * 4;
    const int soff = j / p.Cin, ci = j - soff * p.Cin;
    const bool has_alpha = p.in_alpha != nullptr;
    float4 al = make_float4(0.f, 0.f, 0.f, 0.f), ia = al;
    if (has_alpha) {
        al = __ldg(reinterpret_cast<const float4*>(p.in_alpha + ci));
        ia = __ldg(reinterpret_cast<const float4*>(p.in_inv_alpha + ci));
    }
    const int RSTEP = NT >> lp;
    const int row_limit = p.Tout + (p.Kr - 1) * p.dil;
    const int vrow0 = t0 - p.PLr;
    const float* __restrict__ xcol = xb + ci;
#pragma unroll 1
    for (int r = ptid >> lp; r < R; r += RSTEP * BATCH) {
        float4 v[BATCH];
#pragma unroll
        for (int u = 0; u < BATCH; ++u) {
            const int rr = r + u * RSTEP;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int vrow = vrow0 + rr;
            if (rr < R && vrow < row_limit) {
                const int src = pm.src(vrow * p.vf + soff);
                if (src >= 0) v[u] = __ldg(reinterpret_cast<const float4*>(xcol + (size_t)src * p.ldx));
            }
        }
#pragma unroll
        for (int u = 0; u < BATCH; ++u) {
            const int rr = r + u * RSTEP;
            if (rr < R) {
                float4 x4 = v[u];
                if (has_alpha) x4 = snake4_sel<BF16, INL>(x4, al, ia);   // snake(0) == 0, so padded zeros stay zero
                if constexpr (SINGLE) store_f16_single(x4, pc, rr, Rpad, ahi);
                else if constexpr (F16) split_store_f16(x4, pc, rr, Rpad, ahi, alo);
                else split_store<BF16>(x4, pc, rr, Rpad, ahi, alo);
            }
        }
    }
}

}  // namespace tc

}  // namespace fac
