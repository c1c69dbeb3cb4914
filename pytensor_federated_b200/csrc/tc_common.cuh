// wgmma / TMA / mbarrier PTX wrappers and shared-memory descriptors shared by the tensor-core GLM
// kernels (glm_tc.cu: bf16, glm_fp8.cu: block-scaled fp8).  sm_90a only.
#pragma once
#include <cstdlib>

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include "fed_comm.cuh"
#include "glm_link.cuh"
#include "models.h"

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
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const CUtensorMap* map, int c0, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(smem_u32(bar))
        : "memory");
}
// Plain (non-tensor) bulk copy of `bytes` (a multiple of 16, 16-byte aligned at both ends) into shared memory
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// Named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// v, as a value the compiler cannot prove equal to another copy of it: what is computed from it is recomputed where it
// is used instead of being kept in a register from its first use on
__device__ __forceinline__ int opaque(int v) {
    asm volatile("" : "+r"(v));
    return v;
}

// Register reallocation between warpgroups (setmaxnreg): the calling warpgroup's registers per thread go from `From`
// to `To`, taken from the CTA's pool (inc, which blocks until the pool holds them) or given back to it (dec).  Every
// thread of the warpgroup executes the same instruction, and ptxas allocates the code after it within `To` registers.
template <int From, int To>
__device__ __forceinline__ void setmaxnreg() {
    static_assert(To % 8 == 0 && To >= 24 && To <= 256 && To != From, "setmaxnreg: a multiple of 8 in [24, 256]");
    if constexpr (To > From) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(To));
    else asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(To));
}

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

// Launches `kernel` with `smem` bytes of dynamic shared memory, with programmatic stream serialization when use_pdl()
// (the kernel's theta-independent setup then overlaps the tail of the previous evaluation).  Returns the launch's
// cudaError_t.
template <typename... Params, typename... Args>
int launch_pdl(void (*kernel)(Params...), int grid, int threads, uint32_t smem, cudaStream_t stream, Args... args) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, args...);
    return (int)cudaGetLastError();
}

// The driver's cuTensorMapEncodeTiled, or null when the driver does not have it.
inline PFN_cuTensorMapEncodeTiled encode_tiled() {
    static PFN_cuTensorMapEncodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(p);
    }
    return fn;
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

// Multinomial (softmax) likelihood of one row, family 3.  The row's columns are spread over the four lanes of a
// quad (the lanes sharing lane >> 2); this lane holds NS of them: eta[s] is column s of this lane, chain[s] the
// chain it belongs to (-1: no chain, i.e. a column past K*C) and cls[s] its class.  Per chain, the row maximum m
// and s = sum_c exp(eta_c - m) are reduced over the quad with xor-1 / xor-2 butterflies, which every lane runs
// for every chain below n_chains (a warp-uniform bound): a lane holding no column of a chain contributes -inf / 0.
// Both butterfly steps add or compare the same two values on both partners, so all four lanes get the same bits.
// The chain loops only reduce and hand the result to the lane's columns of that chain; the exponentials, logs and
// reciprocals are evaluated once per column afterwards (NS each, not NS per chain).
// Results: ll[s] = [y == c] (eta_c - m - log s), r[s] = [y == c] - exp(eta_c - m) / s; |r| <= 1.
template <int NS, int MAX_CHAINS>
__device__ __forceinline__ void softmax_loglik(const float (&eta)[NS], const int (&chain)[NS], const float (&cls)[NS],
                                               int n_chains, float y, float (&ll)[NS], float (&r)[NS]) {
    float mx[NS], sm[NS];   // row maximum and sum of exponentials of each column's chain
#pragma unroll
    for (int s = 0; s < NS; ++s) mx[s] = 0.f, sm[s] = 1.f;
#pragma unroll
    for (int k = 0; k < MAX_CHAINS; ++k) {
        if (k >= n_chains) break;
        float m = -INFINITY;
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) m = fmaxf(m, eta[s]);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) mx[s] = m;
    }
    float ex[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) ex[s] = __expf(eta[s] - mx[s]);
#pragma unroll
    for (int k = 0; k < MAX_CHAINS; ++k) {
        if (k >= n_chains) break;
        float sum = 0.f;
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) sum += ex[s];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) sm[s] = sum;
    }
#pragma unroll
    for (int s = 0; s < NS; ++s)
        if (chain[s] >= 0) {
            const bool hit = y == cls[s];
            ll[s] = hit ? (eta[s] - mx[s]) - __logf(sm[s]) : 0.f;
            r[s] = (hit ? 1.f : 0.f) - ex[s] * __fdividef(1.f, sm[s]);
        }
}

// The cumulative-logit terms of one row and chain, with u = z_up = eta - c_y (up: y <= C - 2), l = z_lo =
// eta - c_{y-1} (lo: y >= 1) and the gap d = l - u > 0 (used when both are present):
//   y = 0:      ll = -softplus(u),                                 r_up = -sigmoid(u)
//   y = C - 1:  ll = -softplus(-l),                                r_lo = sigmoid(-l)
//   otherwise:  ll = -softplus(u) - softplus(-l) + log(1 - e^-d),  r_up = -sigmoid(u) - 1 / expm1(d),
//                                                                  r_lo = sigmoid(-l) + 1 / expm1(d)
// softplus, sigmoid and log(1 - e^-d) use expf / log1pf / expm1f, which stay relatively accurate in the tails
// (|c - eta| of 30 and more, gaps of a few hundredths), where __logf(1 + e) would return 0 or log(d) would cancel.
__device__ __forceinline__ void ordinal_terms(float u, float l, float d, bool up, bool lo, float& ll, float& ru, float& rl) {
    const float eu = expf(-fabsf(u)), el = expf(-fabsf(l));
    const float spu = fmaxf(u, 0.f) + log1pf(eu);              // softplus(u)
    const float spl = fmaxf(-l, 0.f) + log1pf(el);             // softplus(-l)
    const float sgu = __fdividef(u >= 0.f ? 1.f : eu, 1.f + eu);   // sigmoid(u)
    const float sgl = __fdividef(l <= 0.f ? 1.f : el, 1.f + el);   // sigmoid(-l)
    const bool mid = up && lo;
    const float lg = d > 0.693147181f ? log1pf(-expf(-d)) : logf(-expm1f(-d));   // log(1 - e^-d)
    const float t = mid ? __frcp_rn(expm1f(d)) : 0.f;          // 0 once expm1 overflows (d > 88)
    ll = ((up ? -spu : 0.f) - (lo ? spl : 0.f)) + (mid ? lg : 0.f);
    ru = -sgu - t;
    rl = sgl + t;
}

// Ordinal (cumulative-logit) likelihood of one row, family 6.  The C - 1 = n_cut cutpoints of chain k are columns
// v = k n_cut + j, and column v holds z_j = eta - c_j (the intercept table row v is intercept - c_j).  As in
// softmax_loglik, the row's columns sit in the four lanes of a quad, this lane holds NS of them (chain[s]: its chain,
// -1 past K n_cut; cut[s]: its cutpoint j).  For label yi (clamped to [0, n_cut]) the row couples only the columns
// up = yi (if yi < n_cut) and lo = yi - 1 (if yi > 0): per chain, their z are summed over the quad with xor-1 / xor-2
// shuffles, which every lane runs for every chain below n_chains (warp-uniform); a lane holding neither column
// adds 0, so the sums are exact and all four lanes get the same bits.  The gap l - u is taken from the intercept
// table, icpt[(k, yi - 1)] - icpt[(k, yi)] of the row's group (icpt_g[v * G]: intercept row v of the row's group): the
// difference of two packed fp32 values, > 0 whenever the host accepted the cutpoints as ordered, and accurate to
// ulp(|intercept - c|) rather than ulp(|z|).  Results: ll[s] = the chain's ll in column min(yi, n_cut - 1) and 0
// elsewhere, r[s] = r_up / r_lo in the up / lo columns and 0 elsewhere.
template <int NS, int MAX_CHAINS>
__device__ __forceinline__ void ordinal_loglik(const float (&z)[NS], const int (&chain)[NS], const int (&cut)[NS],
                                               int n_chains, int n_cut, int yi, const float* icpt_g, int G,
                                               float (&ll)[NS], float (&r)[NS]) {
    const bool up = yi < n_cut, lo = yi > 0;
    const int credit = up ? yi : yi - 1;
#pragma unroll
    for (int s = 0; s < NS; ++s) ll[s] = r[s] = 0.f;
#pragma unroll
    for (int k = 0; k < MAX_CHAINS; ++k) {
        if (k >= n_chains) break;
        float zu = 0.f, zl = 0.f;
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) {
                if (cut[s] == yi) zu = z[s];
                if (cut[s] == yi - 1) zl = z[s];
            }
        zu += __shfl_xor_sync(0xffffffffu, zu, 1);
        zl += __shfl_xor_sync(0xffffffffu, zl, 1);
        zu += __shfl_xor_sync(0xffffffffu, zu, 2);
        zl += __shfl_xor_sync(0xffffffffu, zl, 2);
        const float d = (up && lo) ? icpt_g[(k * n_cut + yi - 1) * G] - icpt_g[(k * n_cut + yi) * G] : 1.f;
        float llk, ru, rl;
        ordinal_terms(zu, zl, d, up, lo, llk, ru, rl);
#pragma unroll
        for (int s = 0; s < NS; ++s)
            if (chain[s] == k) {
                ll[s] = cut[s] == credit ? llk : 0.f;
                r[s] = cut[s] == yi ? ru : (cut[s] == yi - 1 ? rl : 0.f);
            }
    }
}

// Families with a learned dispersion parameter: theta per chain is [intercept[G], beta[P], log_dispersion], and
// the per-chain constants below, derived from log_dispersion at setup (in double), sit in a table of kDispWords
// floats per chain behind the intercepts.
//   family 4, Gaussian with unknown scale, s = log sigma:   ll = -(d / sigma)^2 / 2 - s - log(2 pi) / 2,  d = y - eta
//   family 5, negative binomial (NB2), a = log alpha, mu = exp(eta), var = mu + mu^2 / alpha:
//             ll = lgamma(y + alpha) - lgamma(alpha) + alpha log(alpha / (alpha + mu)) + y log(mu / (alpha + mu))
//             (-lgamma(y + 1) omitted, as in the Poisson family, to which it tends as alpha -> inf)
constexpr int kDispWords = 9;
// table words: Gaussian
constexpr int kDwSinv = 0;     // 1 / sigma = exp(-s)
constexpr int kDwS = 1;        // s
// table words: negative binomial.  lgamma / digamma differences in y are evaluated at alpha' = alpha + m >= 8
// (m = 0 for alpha >= 8) by the Stirling series, and shifted back by the recurrences
//   lgamma(y + alpha) - lgamma(alpha) = [..](alpha') - log prod_{j<m} (y + alpha + j) + log prod_{j<m} (alpha + j),
//   psi(y + alpha) - psi(alpha)       = [..](alpha') - sum_{j<m} 1 / (y + alpha + j) + sum_{j<m} 1 / (alpha + j);
// the sums over alpha alone are per-chain constants.
constexpr int kDwAlpha = 0;    // alpha
constexpr int kDwA = 1;        // a = log alpha
constexpr int kDwM = 2;        // m (0 .. 8)
constexpr int kDwAp = 3;       // alpha'
constexpr int kDwIap = 4;      // 1 / alpha'
constexpr int kDwAph = 5;      // alpha' - 1/2
constexpr int kDwLa = 6;       // log alpha' - log alpha
constexpr int kDwCl = 7;       // log prod_{j<m} (alpha + j) - S(alpha'),  S(z) = 1/(12 z) - 1/(360 z^3) + 1/(1260 z^5)
constexpr int kDwCd = 8;       // sum_{j<m} 1 / (alpha + j) - T(alpha'), T(z) = -1/(2 z) - 1/(12 z^2) + 1/(120 z^4) - 1/(252 z^6)

// The table entries of one chain (family 4 or 5) from its log_dispersion ld.
__device__ inline void dispersion_constants(int family, float ld, float* t) {
    const double l = (double)ld;
    if (family == 4) {
        t[kDwSinv] = (float)exp(-l);   // exactly 1 at s = 0: family 4 then gives family 2's bits
        t[kDwS] = ld;
        return;
    }
    const double alpha = exp(l);
    const int m = alpha < 8.0 ? (int)ceil(8.0 - alpha) : 0;
    const double ap = alpha + m;
    double lp = 0.0, sr = 0.0;
    for (int j = 0; j < m; ++j) {
        lp += log(alpha + j);
        sr += 1.0 / (alpha + j);
    }
    const double i1 = 1.0 / ap, i2 = i1 * i1;
    const double S = i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260)));
    const double T = -0.5 * i1 - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252)));
    t[kDwAlpha] = (float)alpha;
    t[kDwA] = ld;
    t[kDwM] = (float)m;
    t[kDwAp] = (float)ap;
    t[kDwIap] = (float)i1;
    t[kDwAph] = (float)(ap - 0.5);
    t[kDwLa] = (float)(log(ap) - l);
    t[kDwCl] = (float)(lp - S);
    t[kDwCd] = (float)(sr - T);
}

// Family 4 of one row: ll, r = dll/deta and q = dll/ds.  The scaled residual dn = d / sigma goes through family 2's
// expression before s is subtracted, and every sigma operation is exact at sigma = 1, so s = 0 gives family 2's
// ll and r bit for bit.
__device__ __forceinline__ void gaussian_scale_loglik(float y, float eta, const float* t, float& ll, float& r, float& q) {
    const float sinv = t[kDwSinv];
    const float dn = (y - eta) * sinv;
    ll = (-0.5f * dn * dn - 0.918938533204672742f) - t[kDwS];
    r = dn * sinv;
    q = dn * dn - 1.f;
}

// Family 5 of one row: ll, r = dll/deta = y - (alpha + y) sigmoid(x) and
// q = dll/da = alpha [psi(y + alpha) - psi(alpha) - softplus(x)] - r, with x = eta - a.
//   ll = D + y eta - (alpha + y) softplus(x),  D = lgamma(y + alpha) - lgamma(alpha) - y a,
// which takes y log alpha out of both lgamma terms analytically.  At alpha' (see kDwCl):
//   D = (y + alpha' - 1/2) log1p(y / alpha') - y + S(y + alpha') + y (log alpha' - a) - log prod_{j<m} (y + alpha + j)
//       + [log prod_{j<m} (alpha + j) - S(alpha')]
//   psi(y + alpha) - psi(alpha) = log1p(y / alpha') + T(y + alpha') - sum_{j<m} 1 / (y + alpha + j) + [per chain]
// so for alpha >> y nothing of size alpha or y log alpha is ever subtracted: D ~ y (y - 1) / (2 alpha) comes out
// of one FMA with log1p, not of a difference of two lgamma values of size alpha log alpha.  The shift runs a fixed
// 8-step predicated loop (m is per chain), as two products of at most 4 factors (no overflow for y <= 2^24): one
// log and one division each, whatever y is.  softplus and the exponential use log1pf / expf, which are
// relatively accurate at very negative x, where alpha softplus(x) ~ mu.
__device__ __forceinline__ void negbin_loglik(float y, float eta, const float* t, float& ll, float& r, float& q) {
    const float alpha = t[kDwAlpha], ap = t[kDwAp];
    const float x = eta - t[kDwA];
    const float e = expf(-fabsf(x));
    const float sp = fmaxf(x, 0.f) + log1pf(e);
    const float inv = __fdividef(1.f, 1.f + e);
    const float sig = x >= 0.f ? inv : e * inv;
    // recurrence from alpha up to alpha' (m factors y + alpha + j, two products of 4)
    float lp = 0.f, sr = 0.f;
    const int m = (int)t[kDwM];
    if (m > 0) {
        const float ya = y + alpha;
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            float pr = 1.f, nu = 0.f;   // prod f and (sum 1 / f) prod f over this group's factors
#pragma unroll
            for (int j = 4 * g; j < 4 * g + 4; ++j)
                if (j < m) {
                    const float f = ya + (float)j;
                    nu = nu * f + pr;
                    pr = pr * f;
                }
            lp += __logf(pr);
            sr += __fdividef(nu, pr);
        }
    }
    // Stirling series at alpha' >= 8
    const float z = y + ap;
    const float iz = __frcp_rn(z), iz2 = iz * iz;
    const float Sz = iz * (1.f / 12 - iz2 * (1.f / 360 - iz2 * (1.f / 1260)));
    const float Tz = -0.5f * iz - iz2 * (1.f / 12 - iz2 * (1.f / 120 - iz2 * (1.f / 252)));
    const float l1 = log1pf(y * t[kDwIap]);
    const float D = fmaf(y + t[kDwAph], l1, -y) + ((Sz + t[kDwCl]) - lp) + y * t[kDwLa];
    const float dpsi = l1 + ((Tz + t[kDwCd]) - sr);
    const float ay = alpha + y;
    ll = (y * eta - ay * sp) + D;
    r = y - ay * sig;
    q = alpha * (dpsi - sp) - r;
}

// Zero-inflated counts (families 9 and 10), one row of a pair: count predictor eta (offset included), zero logit zeta,
// pi = sigmoid(zeta).  (l, r, q) = the base family's values at eta exactly as the plain family computes them (Poisson:
// link_loglik, NB: negbin_loglik with the chain's table t; both omit -lgamma(y + 1), which is 0 at y = 0, so l is
// log f(0) there), then mixed:
//   y > 0:  ll = l - softplus(zeta),  rc = r,  rz = -sigmoid(zeta),  q unchanged
//   y = 0:  ll = log(e^zeta + e^L0) - softplus(zeta) with L0 = l, d = zeta - L0,  w0 = sigmoid(-d),
//           rc = w0 r,  rz = sigmoid(d) - sigmoid(zeta) = -sigmoid(d) sigmoid(-zeta) expm1(L0),  q = w0 q
// rc = dll/deta, rz = dll/dzeta, q = dll/dlog_alpha.  The product form of rz keeps its relative accuracy as mu -> 0
// (-expm1(L0) ~ mu).  The mixing comes after the base values and in this order, so that at zeta = -120 with
// L0 >= -15 (exp(-|d|) and exp(zeta) underflow to 0, sigmoid(-d) is exactly 1) ll, rc and q are the base family's
// bits and rz is 0.  A NaN y (a masked row) takes the y = 0 branch and is dropped by its weight.
template <bool NB>
__device__ __forceinline__ void zero_inflated_loglik(float y, float eta, float zeta, const float* t, float& ll, float& rc,
                                                     float& rz, float& q) {
    float l, r;
    q = 0.f;
    if constexpr (NB) negbin_loglik(y, eta, t, l, r, q);
    else link_loglik(1, y, eta, l, r);
    const float ez = expf(-fabsf(zeta));
    const float spz = fmaxf(zeta, 0.f) + log1pf(ez);   // softplus(zeta)
    const float iz = __frcp_rn(1.f + ez);
    if (y > 0.f) {
        ll = l - spz;
        rc = r;
        rz = -(zeta >= 0.f ? iz : ez * iz);
    } else {
        const float d = zeta - l;
        const float ed = expf(-fabsf(d));
        ll = (fmaxf(zeta, l) + log1pf(ed)) - spz;
        const float id = __frcp_rn(1.f + ed);
        const float sd = d >= 0.f ? id : ed * id;    // sigmoid(d)
        const float w0 = d >= 0.f ? ed * id : id;    // sigmoid(-d)
        rc = w0 * r;
        q = w0 * q;
        rz = -(sd * (zeta >= 0.f ? ez * iz : iz)) * expm1f(l);
    }
}

// Right-censored survival, accelerated failure time: log T = eta + sigma eps, s = log sigma, z = (log t - eta) / sigma,
// delta = 1 for an event and 0 for a censored row.  Family 7 (Weibull, eps standard minimum-Gumbel, shape 1 / sigma)
// and family 8 (log-normal, eps ~ N(0, 1)) use the Gaussian's table words kDwSinv and kDwS.  The host stores each
// row's time signed in y: +t for an event, -t for a censored row (times are > 0, so the sign bit is free), and the
// kernel takes t = |y|, delta = !signbit(y); log t is a per-row value, computed once per row with logf.
__device__ inline void survival_constants(float ld, float* t) {
    t[kDwSinv] = (float)exp(-(double)ld);
    t[kDwS] = ld;
}

// Family 7 of one row: ll = delta (z - s - log t) - e^z, r = dll/deta = (e^z - delta) / sigma,
// q = dll/ds = z (e^z - delta) - delta.
__device__ __forceinline__ void weibull_loglik(bool event, float lt, float eta, const float* t, float& ll, float& r,
                                               float& q) {
    const float sinv = t[kDwSinv];
    const float z = (lt - eta) * sinv;
    const float ez = expf(z);
    const float d = event ? 1.f : 0.f;
    ll = event ? ((z - ez) - t[kDwS]) - lt : -ez;
    r = (ez - d) * sinv;
    q = z * (ez - d) - d;
}

// Family 8 of one row.  Event: ll = -z^2 / 2 - s - log(2 pi) / 2 - log t, r = z / sigma, q = z^2 - 1.  Censored:
// ll = log Phi(-z), r = lambda / sigma, q = z lambda with the inverse Mills ratio lambda = phi(z) / Phi(-z).  With
// u = z / sqrt(2), Phi(-z) = erfc(u) / 2.  Both signs of u go through one erfcx(a) = e^{a^2} erfc(a) at a = |u|, which
// neither underflows nor loses relative accuracy in the upper tail (fp32 Phi(-z) is subnormal from z ~ 13 and 0 from
// z ~ 14, so log(normcdf(-z)) would give -inf there):
//   u >= 0:  log Phi(-z) = log(erfcx(u) / 2) - u^2,   lambda = sqrt(2 / pi) / erfcx(u)
//   u <  0:  log Phi(-z) = log1p(-h),                 lambda = phi(z) / (1 - h),   h = erfc(-u) / 2 = erfcx(a) e^{-a^2} / 2
__device__ __forceinline__ void lognormal_loglik(bool event, float lt, float eta, const float* t, float& ll, float& r,
                                                 float& q) {
    const float sinv = t[kDwSinv];
    const float z = (lt - eta) * sinv;
    if (event) {
        ll = ((-0.5f * z * z - 0.918938533204672742f) - t[kDwS]) - lt;
        r = z * sinv;
        q = z * z - 1.f;
        return;
    }
    const float u = z * 0.707106781186547524f;
    const float a2 = u * u;
    const float ex = erfcxf(fabsf(u));
    const float g = expf(-a2);                       // e^{-u^2} = sqrt(2 pi) phi(z)
    const float h = 0.5f * ex * g;                   // u < 0: erfc(-u) / 2 = 1 - Phi(-z) <= 1/2
    ll = u >= 0.f ? logf(0.5f * ex) - a2 : log1pf(-h);
    const float lam = u >= 0.f ? 0.797884560802865356f / ex                  // sqrt(2 / pi) / erfcx(u)
                               : 0.398942280401432678f * g / (1.f - h);      // phi(z) / Phi(-z)
    r = lam * sinv;
    q = z * lam;
}

// Positive responses with a log link to the mean (families 11 and 12): mu = e^eta, a = log_dispersion = log of the
// shape (nu for the gamma family, lambda for the inverse Gaussian one), z = log y - eta, log y and 1 / y computed once
// per row.  Per-chain table words, from a at setup in double:
//   gamma:             nu, C(nu) = nu log nu - nu - lgamma(nu), Q(nu) = nu (log nu - psi(nu))
//   inverse Gaussian:  lambda, a / 2 - log(2 pi) / 2
// C and Q come from the Stirling series at nu' = nu + m >= 8, with the shift and series of dispersion_constants (kept
// as a separate copy there: sharing one helper changes the SASS of the negative-binomial instantiations):
//   C(nu) = nu (log nu - log nu') + (1/2 - m) log nu' + m - log(2 pi) / 2 - S(nu') + log prod_{j<m} (nu + j)
//   Q(nu) = nu (log nu - log nu' - T(nu') + sum_{j<m} 1 / (nu + j))
// (S and T as at kDwCl / kDwCd), so that for nu >= 8 (m = 0) nothing of size nu log nu is formed: C -> (log nu -
// log 2 pi) / 2 and Q -> 1/2 as nu grows.
constexpr int kDwShape = 0;    // nu or lambda
constexpr int kDwC0 = 1;       // C(nu), or a / 2 - log(2 pi) / 2
constexpr int kDwQ0 = 2;       // Q(nu) (gamma only)

__device__ inline void positive_constants(int family, float ld, float* t) {
    const double l = (double)ld;
    const double shape = exp(l);
    t[kDwShape] = (float)shape;
    if (family == kGlmInverseGaussian) {
        t[kDwC0] = (float)(0.5 * l - 0.918938533204672742);
        return;
    }
    const int m = shape < 8.0 ? (int)ceil(8.0 - shape) : 0;
    const double sp = shape + m;
    double lp = 0.0, sr = 0.0;
    for (int j = 0; j < m; ++j) {
        lp += log(shape + j);
        sr += 1.0 / (shape + j);
    }
    const double i1 = 1.0 / sp, i2 = i1 * i1;
    const double S = i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260)));
    const double T = -0.5 * i1 - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252)));
    const double lsp = m > 0 ? log(sp) : l;   // log nu'
    const double dl = l - lsp;                  // log nu - log nu', exactly 0 for m = 0
    t[kDwC0] = (float)(shape * dl + (0.5 - m) * lsp + m - 0.918938533204672742 - S + lp);
    t[kDwQ0] = (float)(shape * (dl - T + sr));
}

// Family 11 of one row, lt = log y:
//   ll = nu g(z) + C(nu) - log y,   r = dll/deta = nu expm1(z),   q = dll/da = nu g(z) + Q(nu),   g(z) = 1 + z - e^z.
// g(z) = z - expm1(z) loses about 2 eps / |z| of its relative accuracy near z = 0, which is where the rows sit at a
// large shape (z ~ nu^-1/2), so below |z| = 1/2 it is the series -z^2 (1/2! + z / 3! + ... + z^6 / 8!), whose
// truncation error there is below 2 (1/2)^7 / 9! = 4.3e-8 of g, and expm1(z) = z - g(z) (no cancellation: |g| < |z| / 3).
// From |z| = 1/2 up, e^z - 1 and z - (e^z - 1) lose at most a few eps.  One expf per row and chain.
__device__ __forceinline__ void gamma_loglik(float lt, float eta, const float* t, float& ll, float& r, float& q) {
    const float nu = t[kDwShape];
    const float z = lt - eta;
    const float ez = expf(z);
    float gs = fmaf(z, 1.f / 40320, 1.f / 5040);
    gs = fmaf(z, gs, 1.f / 720);
    gs = fmaf(z, gs, 1.f / 120);
    gs = fmaf(z, gs, 1.f / 24);
    gs = fmaf(z, gs, 1.f / 6);
    gs = fmaf(z, gs, 0.5f);
    gs = -(z * z) * gs;
    const bool small = fabsf(z) < 0.5f;
    const float em = small ? z - gs : ez - 1.f;
    const float g = small ? gs : z - em;
    const float ng = nu * g;
    ll = (ng + t[kDwC0]) - lt;
    r = nu * em;
    q = ng + t[kDwQ0];
}

// Family 12 of one row, lt = log y, iy = 1 / y:
//   ll = a / 2 - log(2 pi) / 2 - (3/2) log y - lambda expm1(z)^2 / (2 y),
//   r = dll/deta = lambda e^-eta expm1(z) = lambda (y - mu) / mu^2,   q = dll/da = 1/2 - lambda expm1(z)^2 / (2 y).
// expm1(z) = y e^-eta - 1 comes from one FMA (the product is not rounded before the subtraction), and expm1(z)^2 / y
// is formed as em (em / y): em / y <= e^-eta, so nothing overflows before the result does.  One expf per row and chain.
__device__ __forceinline__ void inverse_gaussian_loglik(float y, float lt, float iy, float eta, const float* t, float& ll,
                                                        float& r, float& q) {
    const float lam = t[kDwShape];
    const float ei = expf(-eta);
    const float em = fmaf(y, ei, -1.f);
    const float h = 0.5f * lam * (em * (em * iy));
    ll = (fmaf(-1.5f, lt, t[kDwC0])) - h;
    r = lam * (ei * em);
    q = 0.5f - h;
}

// Location-scale regression (families 13 and 14), one row of a pair: mean mu (identity link, offset included) and
// s = log sigma, each its own linear predictor; z = (y - mu) e^-s with e^-s one expf per row and pair.
// Family 13, the Gaussian:  ll = -z^2 / 2 - s - log(2 pi) / 2,  rm = dll/dmu = z e^-s,  rs = dll/ds = z^2 - 1.
// The order of operations is gaussian_scale_loglik's and expf(-0) is exactly 1, so at s = 0 ll and rm are family 2's
// bits.  Once z^2 / 2 overflows, ll is -inf, the correctly rounded value.
__device__ __forceinline__ void location_scale_loglik(float y, float mu, float s, float& ll, float& rm, float& rs) {
    const float sinv = expf(-s);
    const float dn = (y - mu) * sinv;
    ll = (-0.5f * dn * dn - 0.918938533204672742f) - s;
    rm = dn * sinv;
    rs = dn * dn - 1.f;
}

// Family 14, Student-t with nu = e^a degrees of freedom (a = log_dispersion), q = z^2 / nu, p = q / (1 + q):
//   ll = C(nu) - s - (nu + 1) / 2 log1p(q),   rm = (nu + 1) z e^-s / (nu + z^2),   rs = (nu + 1) p - 1,
//   q_a = dll/da = Q(nu) + p / 2 - (nu / 2) h(q),   h(q) = log1p(q) - p,
//   C(nu) = lgamma((nu + 1) / 2) - lgamma(nu / 2) - log(nu pi) / 2,   Q(nu) = (nu / 2) [psi((nu + 1) / 2) - psi(nu / 2)] - 1/2.
// Per-chain table words, from a at setup in double.  Below nu = 1e3, C and Q come from the Stirling series at
// b' = nu / 2 + m >= 8 and a' = b' + 1/2, shifted back by the recurrences (the shift and series of
// dispersion_constants, in a separate copy for the reason given at positive_constants):
//   C = b' log1p(1 / (2 b')) - 1/2 + log(b') / 2 - log(nu pi) / 2 + S(a') - S(b') - sum_{j<m} log1p(1 / (2 (nu / 2 + j)))
//   Q = (nu / 2) [log1p(1 / (2 b')) + T(a') - T(b') + sum_{j<m} (1 / (nu / 2 + j) - 1 / (nu / 2 + j + 1/2))] - 1/2
// (S and T as at kDwCl / kDwCd): no lgamma or psi value is formed, and the largest cancellation, b' log1p(1 / (2 b'))
// against 1/2, costs a factor 4 b' < 2e3 of double precision.  From nu = 1e3 both are their asymptotic series,
//   C = -log(2 pi) / 2 - 1 / (4 nu) + 1 / (24 nu^3) - 1 / (20 nu^5),   Q = 1 / (4 nu) - 1 / (8 nu^3) + 1 / (4 nu^5),
// whose truncation error there is below 1e-20, so no difference of values of size nu log nu is ever taken.
constexpr int kStNu = 0;     // nu
constexpr int kStNp1 = 1;    // nu + 1
constexpr int kStC1 = 2;     // (nu + 1) / nu
constexpr int kStIsq = 3;    // nu^-1/2
constexpr int kStHn = 4;     // nu / 2
constexpr int kStC = 5;      // C(nu)
constexpr int kStQ = 6;      // Q(nu)

__device__ inline void student_t_constants(float ld, float* t) {
    const double l = (double)ld;
    const double nu = exp(l);
    double C, Q;
    if (nu < 1e3) {
        const double b = 0.5 * nu;
        const int m = b < 8.0 ? (int)ceil(8.0 - b) : 0;
        const double bp = b + m, ap = bp + 0.5;
        double ls = 0.0, rs = 0.0;
        for (int j = 0; j < m; ++j) {
            ls += log1p(0.5 / (b + j));
            rs += 1.0 / (b + j) - 1.0 / (b + j + 0.5);
        }
        const auto S = [](double z) {
            const double i1 = 1.0 / z, i2 = i1 * i1;
            return i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260)));
        };
        const auto T = [](double z) {
            const double i1 = 1.0 / z, i2 = i1 * i1;
            return -0.5 * i1 - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252)));
        };
        const double l1 = log1p(0.5 / bp);
        C = (bp * l1 - 0.5) + 0.5 * (log(bp) - l - 1.1447298858494002) + (S(ap) - S(bp)) - ls;   // log pi
        Q = b * (l1 + (T(ap) - T(bp)) + rs) - 0.5;
    } else {
        const double x = 1.0 / nu, x2 = x * x;
        C = -0.918938533204672742 - x * (0.25 - x2 * (1.0 / 24 - x2 * (1.0 / 20)));
        Q = x * (0.25 - x2 * (0.125 - x2 * 0.25));
    }
    t[kStNu] = (float)nu;
    t[kStNp1] = (float)(nu + 1.0);
    t[kStC1] = (float)((nu + 1.0) / nu);
    t[kStIsq] = (float)(1.0 / sqrt(nu));
    t[kStHn] = (float)(0.5 * nu);
    t[kStC] = (float)C;
    t[kStQ] = (float)Q;
}

// Family 14 of one row (see student_t_constants), with u = |z| nu^-1/2 = sqrt(q):
// - q < 2^24 (u < 2^12): log1p(q), p = q / (1 + q) and z / (nu + z^2) = (z / (1 + q)) / nu directly;
// - q >= 2^24, where z^2 may overflow (|z| up to ~1e30 and beyond stays finite): with 1 / q = (nu / z) / z,
//   log1p(q) = 2 log u + log1p(1 / q), where log1p(1 / q) = 1 / q to within 2^-49, p = 1 / (1 + 1 / q) and
//   z / (nu + z^2) = (1 / z) p, so rm -> 0 as |z| grows (bounded influence) and nothing overflows.
// log u is taken as log1p(u - 1) (u - 1 is exact for u >= 2^12), so a row costs one log1p whichever branch it takes.
// h(q) = log1p(q) - p loses about 2 eps / q to cancellation for small q, where the rows sit at a large nu (q ~ 1 / nu),
// so below q = 1/4 (p < 1/5) it is the series of -log1p(-p) - p = sum_{k>=2} p^k / k, all terms positive, to k = 12:
// the truncation error is below 2 (1/5)^11 / 13 / (4/5) < 4e-9 of h.  From q = 1/4 up the difference loses < 8 eps.
__device__ __forceinline__ void student_t_loglik(float y, float mu, float s, const float* t, float& ll, float& rm,
                                                 float& rs, float& qa) {
    const float sinv = expf(-s);
    const float z = (y - mu) * sinv;
    const float u = fabsf(z) * t[kStIsq];
    const float q = u * u;
    const bool big = u >= 4096.f;
    const float rz = __frcp_rn(z);
    const float iq = (t[kStNu] * rz) * rz;                 // 1 / q (big rows)
    const float d = __frcp_rn(1.f + (big ? iq : q));       // big: p, else 1 / (1 + q)
    const float p = big ? d : q * d;
    const float lg = log1pf(big ? u - 1.f : q);
    const float L = big ? fmaf(2.f, lg, iq) : lg;          // log1p(q)
    float hs = fmaf(p, 1.f / 12, 1.f / 11);
    hs = fmaf(p, hs, 1.f / 10);
    hs = fmaf(p, hs, 1.f / 9);
    hs = fmaf(p, hs, 1.f / 8);
    hs = fmaf(p, hs, 1.f / 7);
    hs = fmaf(p, hs, 1.f / 6);
    hs = fmaf(p, hs, 1.f / 5);
    hs = fmaf(p, hs, 1.f / 4);
    hs = fmaf(p, hs, 1.f / 3);
    hs = fmaf(p, hs, 0.5f);
    const float h = q < 0.25f ? (p * p) * hs : L - p;
    const float np1 = t[kStNp1];
    ll = fmaf(-0.5f * np1, L, t[kStC]) - s;
    rm = (big ? np1 * (rz * p) : t[kStC1] * (z * d)) * sinv;
    rs = fmaf(np1, p, -1.f);
    qa = fmaf(-t[kStHn], h, fmaf(0.5f, p, t[kStQ]));
}

// Beta regression (family 15): y in (0, 1), mu = sigmoid(eta), phi = e^a the precision (a = log_dispersion),
// A = mu phi, B = (1 - mu) phi, y ~ Beta(A, B).  With the Stirling tail S(z) = lgamma(z) - [(z - 1/2) log z - z +
// log(2 pi) / 2], tau(z) = psi(z) - log z and the Bernoulli divergence KL = mu log(mu / y) + (1 - mu) log((1 - mu) /
// (1 - y)) >= 0, the density is grouped so that nothing of size phi log phi is formed:
//   ll = C(phi) + (log mu + log(1 - mu)) / 2 - log y - log(1 - y) - phi KL - S(A) - S(B),
//   r  = dll/deta = phi mu (1 - mu) (logit y - logit mu) - (1 - mu) A tau(A) + mu B tau(B),
//   q  = dll/da   = Q(phi) - phi KL - A tau(A) - B tau(B),
// C(phi) = (a - log 2 pi) / 2 + S(phi) and Q(phi) = phi tau(phi) per chain, from a at setup in double: below phi = 8
// through the recurrence to phi' = phi + m >= 8, from 8 up as their asymptotic series, so Q -> -1/2 is never the
// difference of values of size phi.
constexpr int kBtPhi = 0;    // phi
constexpr int kBtC = 1;      // C(phi)
constexpr int kBtQ = 2;      // Q(phi)
constexpr int kBtA = 3;      // a = log phi

__device__ inline void beta_constants(float ld, float* t) {
    const double l = (double)ld;
    const double phi = exp(l);
    double S, Q;
    if (phi < 8.0) {
        const int m = (int)ceil(8.0 - phi);
        const double pp = phi + m;
        double lp = 0.0, sr = 0.0;   // the factors phi + j, j = 1 .. m - 1 (j = 0 is taken through l = log phi)
        for (int j = 1; j < m; ++j) {
            lp += log(phi + j);
            sr += 1.0 / (phi + j);
        }
        const double i1 = 1.0 / pp, i2 = i1 * i1, lpp = log(pp);
        const double Sp = i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260 - i2 * (1.0 / 1680))));
        const double Tp = -0.5 * i1 - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240))));
        S = Sp + (pp - 0.5) * lpp - (phi + 0.5) * l - m - lp;
        Q = phi * (Tp + (lpp - l) - sr) - 1.0;
    } else {
        const double i1 = 1.0 / phi, i2 = i1 * i1;
        S = i1 * (1.0 / 12 - i2 * (1.0 / 360 - i2 * (1.0 / 1260 - i2 * (1.0 / 1680))));
        Q = -0.5 - i1 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240))));
    }
    t[kBtPhi] = (float)phi;
    t[kBtC] = (float)(0.5 * (l - 1.83787706640934548) + S);   // log 2 pi
    t[kBtQ] = (float)Q;
    t[kBtA] = ld;
}

// S(z) and z tau(z) of one z > 0 that changes from row to row, lz = log z given (z = A or B may underflow where its
// logarithm does not).  Below z = 8 the argument is shifted to z' = z + m, m = ceil(8 - z) in 1 .. 8:
//   S(z) = S(z') + (z' - 1/2) log z' - (z + 1/2) log z - m - log prod_{j=1}^{m-1} (z + j),
//   z tau(z) = z [T(z') + log z' - log z - sum_{j=1}^{m-1} 1 / (z + j)] - 1,
// with the j = 0 factor taken analytically (its log is lz, z / z = 1), so a z near 0 costs nothing in accuracy.
// The factors run as a fixed, predicated loop of 7 steps in two products of at most 4 (no loop length depends on
// the row, and the products stay below 16^4): one __logf and one division each.  S and T are the series of kDwCl /
// kDwCd at z' >= 8.
__device__ __forceinline__ void beta_tails(float z, float lz, float& S, float& zt) {
    const int m = z < 8.f ? (int)ceilf(8.f - z) : 0;
    float lp = 0.f, sr = 0.f;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        float pr = 1.f, nu = 0.f;   // prod f and (sum 1 / f) prod f over this group's factors
#pragma unroll
        for (int j = 4 * g + 1; j < 4 * g + 5 && j < 8; ++j)
            if (j < m) {
                const float f = z + (float)j;
                nu = fmaf(nu, f, pr);
                pr = pr * f;
            }
        lp += __logf(pr);
        sr += __fdividef(nu, pr);
    }
    const float zp = z + (float)m;
    const float iz = __frcp_rn(zp), iz2 = iz * iz;
    const float Sz = iz * (1.f / 12 - iz2 * (1.f / 360 - iz2 * (1.f / 1260)));
    const float Tz = -0.5f * iz - iz2 * (1.f / 12 - iz2 * (1.f / 120 - iz2 * (1.f / 252)));
    const float lzp = logf(zp);
    const bool shift = m > 0;
    S = shift ? Sz + ((fmaf(zp - 0.5f, lzp, -(float)m) - lp) - (z + 0.5f) * lz) : Sz;
    zt = shift ? fmaf(z, (Tz - sr) + (lzp - lz), -1.f) : z * Tz;
}

// k(x) = x - log1p(x) >= 0 for |x| < 1/2 from s = x / (2 + x) (log1p(x) = 2 atanh(s), x - 2 s = x s):
//   k(x) = x s - 2 s^3 (1/3 + s^2 / 5 + ... + s^12 / 15),
// no cancellation (2 s^3 / 3 < x s / 16 for x > 0; both terms >= 0 for x < 0) and a truncation error below 5e-9 of
// k at |s| <= 1/3, where x - log1pf(x) would lose about 2 eps / |x| of k.
__device__ __forceinline__ float beta_kl_series(float x) {
    const float s = x * __frcp_rn(2.f + x), s2 = s * s;
    float p = fmaf(s2, 1.f / 15, 1.f / 13);
    p = fmaf(s2, p, 1.f / 11);
    p = fmaf(s2, p, 1.f / 9);
    p = fmaf(s2, p, 1.f / 7);
    p = fmaf(s2, p, 1.f / 5);
    p = fmaf(s2, p, 1.f / 3);
    return fmaf(x, s, -2.f * (s * s2) * p);
}

// Family 15 of one row (see beta_constants), ly = log y and l1y = log(1 - y) computed once per row.  mu and 1 - mu
// both come from e = exp(-|eta|) (1 - mu is never 1 - mu rounded), and so do log mu = -softplus(-eta), log(1 - mu)
// and 1 / mu, 1 / (1 - mu).  The relative differences u = (y - mu) / mu and v = (mu - y) / (1 - mu) give
//   logit y - logit mu = log1p(u) - log1p(v),   phi KL = A k(u) + B k(v)   (mu u + (1 - mu) v = 0),
// so neither cancels at y ~ mu, where the rows sit at a large phi (|y - mu| ~ phi^-1/2): below |x| = 1/2, k is
// beta_kl_series and log1p(x) = x - k(x); from 1/2 up, log1p(u) = log y - log mu (and log1p(v) = log(1 - y) -
// log(1 - mu)), which stays finite where 1 + u loses all its digits, and A k(u) = phi (y - mu) - A log1p(u).  y - mu is
// formed as (1 - mu) - (1 - y) for mu >= 1/2, exact where the two are close.  log A = log mu + a is never log of A.
__device__ __forceinline__ void beta_loglik(float y, float ly, float l1y, float eta, const float* t, float& ll, float& r,
                                            float& q) {
    const float phi = t[kBtPhi];
    const float e = expf(-fabsf(eta));
    const float l1e = log1pf(e);
    const float inv = __frcp_rn(1.f + e);
    const bool pos = eta >= 0.f;
    const float mu = pos ? inv : e * inv, nmu = pos ? e * inv : inv;              // mu, 1 - mu
    const float lmu = pos ? -l1e : eta - l1e, l1mu = pos ? -eta - l1e : -l1e;      // log mu, log(1 - mu)
    const float d = pos ? nmu - (1.f - y) : y - mu;                                 // y - mu
    const float pd = phi * d;
    // the terms that do not involve the tails first, each side (u, then v) finished before the next starts, and each
    // tail folded into ll, r and q as soon as it is known: few values stay live at once
    float kl, dlg;   // phi KL, logit y - logit mu
    {
        const float A = mu * phi;
        const float u = d * (pos ? 1.f + e : 1.f + __frcp_rn(e));                   // (y - mu) / mu
        const bool su = fabsf(u) < 0.5f;
        const float ku = beta_kl_series(u);
        const float lu = su ? u - ku : ly - lmu;                                     // log1p(u)
        kl = su ? A * ku : fmaf(-A, lu, pd);
        dlg = lu;
    }
    {
        const float B = nmu * phi;
        const float v = -d * (pos ? 1.f + __frcp_rn(e) : 1.f + e);                  // (mu - y) / (1 - mu)
        const bool sv = fabsf(v) < 0.5f;
        const float kv = beta_kl_series(v);
        const float lv = sv ? v - kv : l1y - l1mu;                                   // log1p(v)
        kl += sv ? B * kv : fmaf(-B, lv, -pd);
        dlg -= lv;
    }
    ll = (fmaf(0.5f, lmu + l1mu, t[kBtC]) - (ly + l1y)) - kl;
    r = (mu * phi) * nmu * dlg;
    q = t[kBtQ] - kl;
    float S, zt;
    beta_tails(mu * phi, lmu + t[kBtA], S, zt);
    ll -= S;
    r = fmaf(-nmu, zt, r);
    q -= zt;
    beta_tails(nmu * phi, l1mu + t[kBtA], S, zt);
    ll -= S;
    r = fmaf(mu, zt, r);
    q -= zt;
}


}  // namespace tc
