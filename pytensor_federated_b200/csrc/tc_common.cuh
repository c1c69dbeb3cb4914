// wgmma / TMA / mbarrier PTX wrappers and shared-memory descriptors shared by the tensor-core GLM
// kernels (glm_tc.cu: bf16, glm_fp8.cu: block-scaled fp8).  sm_90a only.
#pragma once
#include <cstdlib>

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "fed_comm.cuh"

namespace tc {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// CTA-wide "the mbarrier pipeline stalled" flag.  A wait that exceeds 4 s raises it instead of trapping (a
// trap poisons the whole CUDA context: engine, torch and all); once it is up every wait returns at once, so the
// roles run off the end of their loops, the CTA reports B200FED_ERR_PIPELINE through fed::epilogue and the host
// raises an ordinary exception with the context intact.  Results of such a launch are garbage by definition.
__device__ __forceinline__ volatile int* pipeline_fault() {
    __shared__ int fault;
    return &fault;
}
// Bounded wait: a pipeline bug must surface as an error status, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const unsigned long long t0 = fed::globaltimer();
    volatile int* fault = pipeline_fault();
    while (!mbar_try_wait(bar, parity)) {
        if (*fault) return;
        if (fed::globaltimer() - t0 > 4000000000ull) {
            *fault = 1;
            return;
        }
    }
}
// One lane of a fully active warp (the role loops stay warp-uniform; only the issue is predicated, so the
// compiler keeps descriptors and addresses in uniform registers instead of a per-instruction waterfall).
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy stores to shared memory -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// Named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// ------------------------------------------------------------------ wgmma (sm_90a)
// Warpgroup MMA: 128 threads (4 consecutive warps, the first a multiple of 4) issue together; the fp32
// accumulator of an m64nN tile lives in registers, N / 2 per thread: d[4j + 2h + e] = (row 16 w + lane / 4 + 8 h,
// column 8 j + 2 (lane % 4) + e) for warp w of the group.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across wgmma issue and wait.
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// bf16 x bf16 -> fp32, K = 16.  TA / TB: 0 = K-major, 1 = MN-major operand in shared memory.
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    static_assert(N == 8 || N == 16 || N == 24 || N == 32 || N == 48, "instantiated widths");
    if constexpr (N == 8) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 16) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 24) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, %12, %13, p, 1, 1, %15, %16;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
            : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 32) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 48) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
    }
}

// e4m3 x e4m3 -> fp32, K = 32 (both operands K-major: sm_90 has no transposed 8-bit operands).
template <int N>
__device__ __forceinline__ void wgmma_e4m3(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    static_assert(N == 32 || N == 40, "instantiated widths");
    if constexpr (N == 32) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"(scale_d));
    } else if constexpr (N == 40) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n40k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
            : "l"(adesc), "l"(bdesc), "r"(scale_d));
    }
}

// ------------------------------------------------------------------ descriptors
// Shared-memory matrix descriptor (sm_90): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) |
// layout [62,64) (0 = no swizzle, 1 = 128B swizzle).  K-major: SBO = stride between 8-row groups along M / N,
// LBO = stride between the two core matrices along K (no swizzle only).  MN-major 128B swizzle: LBO = stride
// between 64-element spans along M / N, SBO = stride between 8-row groups along K.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle128) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)(swizzle128 ? 1 : 0) << 62;
    return d;
}

// Programmatic dependent launch for back-to-back evaluations (B200FED_NO_PDL=1 disables it).
inline bool use_pdl() {
    static const bool on = [] {
        const char* v = getenv("B200FED_NO_PDL");
        return !(v && *v && *v != '0');
    }();
    return on;
}

// Index + phase bit of an n-deep circular buffer, advanced without division (the single-thread
// TMA / MMA issue loops are latency chains: a 64-bit `it % n`, `it / n` pair costs ~100 instructions).
struct Ring {
    int idx = 0;
    uint32_t phase = 0;
    __host__ __device__ __forceinline__ void advance(int n) {
        if (++idx == n) {
            idx = 0;
            phase ^= 1u;
        }
    }
};

// (hi, lo) += x on a pair that only this thread touches during the launch
__device__ __forceinline__ void dd_accumulate(double* slot, double x) {
    double2 cur = *reinterpret_cast<double2*>(slot);
    fed::dd_add(cur.x, cur.y, x, 0.0);
    *reinterpret_cast<double2*>(slot) = cur;
}

__device__ __forceinline__ void link_loglik(int family, float y, float eta, float& ll, float& r) {
    if (family == 0) {
        const float e = __expf(-fabsf(eta));
        const float sp = fmaxf(eta, 0.f) + __logf(1.f + e);
        const float inv = __fdividef(1.f, 1.f + e);
        const float p = eta >= 0.f ? inv : e * inv;
        ll = y * eta - sp;
        r = y - p;
    } else if (family == 1) {
        const float mu = __expf(eta);
        ll = y * eta - mu;
        r = y - mu;
    } else {
        const float d = y - eta;
        ll = -0.5f * d * d - 0.918938533204672742f;
        r = d;
    }
}


}  // namespace tc
