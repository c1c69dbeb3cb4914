// General-shape GLM kernel: any feature count P <= 1024, any row stride, bf16 or fp32 design matrix.
//
// The fast kernels have shape constraints (glm_tc.cu: P % 128 == 0, bf16; glm_simt.cu: P % 8 == 0,
// 16-byte aligned rows, bf16).  This one has none: a warp takes one row at a time, lane l owns the
// features l, l+32, l+64, ... (coalesced scalar loads), forms the dot product with a shuffle
// reduction and accumulates X^T r from the registers that still hold the row — still a single pass
// over X.  It is the explicit, documented fallback of the fused path (SURVEY.md §7.4: "make the
// fallback explicit, not silent"); arbitrary Python compute functions use the gRPC / local-node path.
#include <cuda_bf16.h>
#include "fed_comm.cuh"
#include "glm_link.cuh"
#include "models.h"
#ifdef B200FED_SNIPPET_HEADER
#include B200FED_SNIPPET_HEADER   // defines B200FED_CUSTOM_LINK (models/custom.py, build.py)
#endif

namespace {

constexpr int kWarpsG = 8;

__device__ __forceinline__ float load_elem(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float load_elem(const float* p) { return __ldg(p); }

#ifdef B200FED_CUSTOM_LINK
// User-supplied likelihood (see models/custom.py): the macro body assigns `ll` (log-likelihood of one
// observation) and `r` (d ll / d eta) from `y` and `eta`.  Compiled into its own shared object.
__device__ __forceinline__ void link_loglik_g(int family, float y, float eta, float& ll, float& r) {
    (void)family;
    B200FED_CUSTOM_LINK
}
#else
__device__ __forceinline__ void link_loglik_g(int family, float y, float eta, float& ll, float& r) {
    link_loglik(family, y, eta, ll, r);
}
#endif
#ifndef B200FED_GENERIC_ENTRY
#define B200FED_GENERIC_ENTRY b200_launch_glm_generic
#endif

template <typename T, int J>  // J = ceil(P / 32) rounded up to 8 / 16 / 32
__global__ void __launch_bounds__(kWarpsG * 32, 2)
fed_glm_generic_kernel(FedComm comm, const GlmSegment* __restrict__ segs, GlmParams prm) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int P = prm.n_features;
    const int G = prm.n_groups;
    float* theta = reinterpret_cast<float*>(smem_raw);                 // [G + P]
    float* g_red = theta + ((comm.n_theta + 3) & ~3);                  // [kWarpsG][J * 32]
    unsigned long long* gi_acc = reinterpret_cast<unsigned long long*>(g_red + kWarpsG * J * 32);  // fixed point
    double* red = reinterpret_cast<double*>(gi_acc + ((G + 1) & ~1));

    fed::Prologue pro = fed::prologue(comm, theta);
    if (!pro.stop && !pro.timed_out) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int i = threadIdx.x; i < G; i += blockDim.x) gi_acc[i] = 0ull;
        // Per-node output blocks (prm.n_out > 1, GlmSegment::out_group): a warp's contiguous row range may cross
        // node boundaries, so its sums are flushed at every boundary (and at the end) into this CTA's row of
        // the partial array, used as 40.24 fixed-point accumulators — integer atomics are associative, the result
        // does not depend on the order of the warps — and converted to doubles in place before the reduction.
        const int NOUT = prm.n_out;
        const int NV1 = 1 + G + P;
        double* out = comm.cta_partials + (size_t)blockIdx.x * comm.n_vals;
        unsigned long long* fx = reinterpret_cast<unsigned long long*>(out);
        if (NOUT > 1)
            for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) fx[i] = 0ull;
        __syncthreads();
        float beta[J], g[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int f = lane + 32 * j;
            beta[j] = f < P ? theta[G + f] : 0.f;
            g[j] = 0.f;
        }
        double ll_total = 0.0;
        float ll_acc = 0.f, gi = 0.f;
        int flush = 0;
        // contiguous range of rows (the segment list uses 8-row "tiles" like the SIMT kernel)
        const long long W = (long long)gridDim.x * kWarpsG;
        const long long gw = (long long)blockIdx.x * kWarpsG + warp;
        const long long T8 = prm.total_tiles;
        long long b = gw * T8 / W;
        const long long b_end = (gw + 1) * T8 / W;
        int s = 0;
        while (s + 1 < prm.n_segments && segs[s + 1].first_tile <= b) ++s;
        GlmSegment seg = segs[s];
        float icpt = theta[seg.group];
        for (; b < b_end; ++b) {
            while (b >= seg.first_tile + ((seg.n_rows + 7) / 8)) {
                if (lane == 0) fed::fix_add(NOUT > 1 ? &fx[seg.out_group * NV1 + 1 + seg.group] : &gi_acc[seg.group], (double)gi);
                gi = 0.f;
                const int og = seg.out_group;
                seg = segs[++s];
                icpt = theta[seg.group];
                if (NOUT > 1 && seg.out_group != og) {   // node boundary: flush this warp's sums into block og
#pragma unroll
                    for (int j = 0; j < J; ++j) {
                        const int f = lane + 32 * j;
                        if (f < P) fed::fix_add(&fx[og * NV1 + 1 + G + f], (double)g[j]);
                        g[j] = 0.f;
                    }
                    if (lane == 0) fed::fix_add(&fx[og * NV1], ll_total + (double)ll_acc);
                    ll_total = 0.0;
                    ll_acc = 0.f;
                    flush = 0;
                }
            }
            const T* Xs = reinterpret_cast<const T*>(seg.X);
            const long long r0 = (b - seg.first_tile) * 8;
            for (int rr = 0; rr < 8; ++rr) {
                const long long row = r0 + rr;
                if (row >= seg.n_rows) break;
                float x[J];
                float p = 0.f;
#pragma unroll
                for (int j = 0; j < J; ++j) {
                    const int f = lane + 32 * j;
                    x[j] = f < P ? load_elem(Xs + row * (long long)prm.ld + f) : 0.f;
                    p = fmaf(x[j], beta[j], p);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
                float ll, r;
                // per-row offset / weight (null: absent, uniform per segment) around the likelihood, custom ones
                // included; rounded on their own, so w = 1, o = 0 gives the bits of the plain model, and a zero weight
                // selects 0 over a non-finite y or offset
                float eta = p + icpt;
                if (seg.offset) eta = __fadd_rn(eta, __ldg(seg.offset + row));
                link_loglik_g(prm.family, __ldg(seg.y + row), eta, ll, r);
                if (seg.weight) {
                    const float wt = __ldg(seg.weight + row);
                    apply_weight(wt, ll);
                    apply_weight(wt, r);
                }
#pragma unroll
                for (int j = 0; j < J; ++j) g[j] = fmaf(r, x[j], g[j]);
                if (lane == 0) {
                    ll_acc += ll;
                    gi += r;
                }
            }
            if (++flush == 64) {
                ll_total += (double)ll_acc;
                ll_acc = 0.f;
                flush = 0;
            }
        }
        ll_total += (double)ll_acc;
        if (NOUT > 1) {
            if (b_end > gw * T8 / W) {
                const int og = seg.out_group;
#pragma unroll
                for (int j = 0; j < J; ++j) {
                    const int f = lane + 32 * j;
                    if (f < P) fed::fix_add(&fx[og * NV1 + 1 + G + f], (double)g[j]);
                }
                if (lane == 0) {
                    fed::fix_add(&fx[og * NV1], ll_total);
                    fed::fix_add(&fx[og * NV1 + 1 + seg.group], (double)gi);
                }
            }
            __syncthreads();
            for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) out[i] = fed::fix_get(__ldcg(&fx[i]));
        } else {
        if (lane == 0 && b_end > gw * T8 / W) fed::fix_add(&gi_acc[seg.group], (double)gi);
#pragma unroll
        for (int j = 0; j < J; ++j) g_red[warp * (J * 32) + lane + 32 * j] = g[j];
        const double ll_block = fed::block_sum(ll_total, red);
        if (threadIdx.x == 0) out[0] = ll_block;
        for (int i = threadIdx.x; i < G; i += blockDim.x) out[1 + i] = fed::fix_get(gi_acc[i]);
        for (int f = threadIdx.x; f < P; f += blockDim.x) {
            double sum = 0.0;
#pragma unroll
            for (int w = 0; w < kWarpsG; ++w) sum += (double)g_red[w * (J * 32) + f];
            out[1 + G + f] = sum;
        }
        }
    }
    fed::epilogue(comm, pro, 0ull);
}

template <typename T, int J>
int launch_generic(const FedComm* comm, const GlmSegment* segs, const GlmParams* prm, int grid, cudaStream_t stream) {
    const size_t smem = (size_t)((comm->n_theta + 3) & ~3) * 4 + (size_t)kWarpsG * J * 32 * 4 +
                        (size_t)((prm->n_groups + 1) & ~1) * 8 + 32 * 8;
    cudaFuncSetAttribute(fed_glm_generic_kernel<T, J>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    fed_glm_generic_kernel<T, J><<<grid, kWarpsG * 32, smem, stream>>>(*comm, segs, *prm);
    return (int)cudaGetLastError();
}

}  // namespace

// elem_bytes: 2 = bf16, 4 = fp32
extern "C" int B200FED_GENERIC_ENTRY(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, int elem_bytes,
                                       int grid, cudaStream_t stream) {
    if (prm->n_chains != 1 || prm->n_features < 1 || prm->n_features > 1024) return -1;
    const int j = (prm->n_features + 31) / 32;
    if (elem_bytes == 2) {
        if (j <= 8) return launch_generic<__nv_bfloat16, 8>(comm, segs_dev, prm, grid, stream);
        if (j <= 16) return launch_generic<__nv_bfloat16, 16>(comm, segs_dev, prm, grid, stream);
        return launch_generic<__nv_bfloat16, 32>(comm, segs_dev, prm, grid, stream);
    }
    if (elem_bytes == 4) {
        if (j <= 8) return launch_generic<float, 8>(comm, segs_dev, prm, grid, stream);
        if (j <= 16) return launch_generic<float, 16>(comm, segs_dev, prm, grid, stream);
        return launch_generic<float, 32>(comm, segs_dev, prm, grid, stream);
    }
    return -1;
}
