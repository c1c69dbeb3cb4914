// Federated GLM log-likelihood + gradient, single pass over a bf16 design matrix (SIMT path).
//
//   eta = intercept[group] + X beta (+ offset) ;  LL = sum w ll(y, eta) ;  r = w dll/deta
//   dLL/dintercept[g] = sum_{rows of g} r ;  dLL/dbeta = X^T r
//
// X is read from HBM exactly once per evaluation: a warp loads 8 rows (one 16-byte
// LDG per lane per row per 256-feature chunk), forms the 8 dot products with a
// transposing butterfly (9 shuffles instead of 40), evaluates link/likelihood in-lane
// and immediately accumulates X^T r from the registers that still hold the rows.
// A stock two-pass implementation (X @ beta, then X.T @ r) moves the matrix twice.
//
// This kernel evaluates one parameter vector per launch and is the numerics reference /
// general-shape path; glm_tc.cu is the wgmma + TMA version that batches MCMC chains.
// There is no GLM in the reference repository; the workload comes from
// BASELINE.json ("federated logistic GLM, 10M rows x 256 features per shard").
#include <cuda_bf16.h>
#include "fed_comm.cuh"
#include "glm_link.cuh"
#include "models.h"

namespace {

constexpr int kWarps = 8;
constexpr int kBatch = 8;  // rows per warp iteration

__device__ __forceinline__ uint4 ldg_stream(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int NCH>
__global__ void __launch_bounds__(kWarps * 32, (NCH == 1 ? 2 : 1))
fed_glm_simt_kernel(FedComm comm, const GlmSegment* __restrict__ segs, GlmParams prm) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int P = prm.n_features;
    const int G = prm.n_groups;
    float* theta = reinterpret_cast<float*>(smem_raw);                         // [G + P]
    float* g_red = theta + ((comm.n_theta + 3) & ~3);                          // [kWarps][P]
    unsigned long long* gi_acc = reinterpret_cast<unsigned long long*>(g_red + kWarps * NCH * 256);  // [G] fixed point
    double* red = reinterpret_cast<double*>(gi_acc + ((G + 1) & ~1));                                      // [32]

    fed::Prologue pro = fed::prologue(comm, theta);
    if (!pro.stop && !pro.timed_out) {
        const int lane = threadIdx.x & 31;
        const int warp = threadIdx.x >> 5;
        for (int i = threadIdx.x; i < G; i += blockDim.x) gi_acc[i] = 0ull;
        // Per-node output blocks (prm.n_out > 1): see csrc/glm_generic.cu — warps flush their sums at node
        // boundaries into this CTA's row of the partial array, used as fixed-point accumulators.
        const int NOUT = prm.n_out;
        const int NV1 = 1 + G + P;
        double* out = comm.cta_partials + (size_t)blockIdx.x * comm.n_vals;
        unsigned long long* fx = reinterpret_cast<unsigned long long*>(out);
        if (NOUT > 1)
            for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) fx[i] = 0ull;
        __syncthreads();

        // this lane's slice of beta
        float beta[NCH][8];
        bool lane_on[NCH];
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            const int f0 = c * 256 + lane * 8;
            lane_on[c] = f0 < P;
#pragma unroll
            for (int k = 0; k < 8; ++k) beta[c][k] = lane_on[c] ? theta[G + f0 + k] : 0.f;
        }
        float g[NCH][8];
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int k = 0; k < 8; ++k) g[c][k] = 0.f;
        double ll_total = 0.0;   // replicated x4 across the lanes of a row group
        float ll_acc = 0.f, gi = 0.f;
        int flush_count = 0;

        // contiguous range of 8-row batches for this warp
        const long long W = (long long)gridDim.x * kWarps;
        const long long gw = (long long)blockIdx.x * kWarps + warp;
        const long long T = prm.total_tiles;
        long long b = gw * T / W;
        const long long b_end = (gw + 1) * T / W;

        int s = 0;
        while (s + 1 < prm.n_segments && segs[s + 1].first_tile <= b) ++s;
        GlmSegment seg = segs[s];
        float icpt = theta[seg.group];
        const int jrow = lane >> 2;  // the row of the batch whose eta ends up in this lane

        for (; b < b_end; ++b) {
            while (b >= seg.first_tile + ((seg.n_rows + kBatch - 1) / kBatch)) {
                // segment switch: flush the intercept gradient of the finished group
                gi = warp_sum(gi);  // every row's r sits in 4 lanes -> x0.25
                if (lane == 0) fed::fix_add(NOUT > 1 ? &fx[seg.out_group * NV1 + 1 + seg.group] : &gi_acc[seg.group], (double)gi * 0.25);
                gi = 0.f;
                const int og = seg.out_group;
                seg = segs[++s];
                icpt = theta[seg.group];
                if (NOUT > 1 && seg.out_group != og) {   // node boundary: flush this warp's sums into block og
#pragma unroll
                    for (int c = 0; c < NCH; ++c)
#pragma unroll
                        for (int k = 0; k < 8; ++k) {
                            if (lane_on[c]) fed::fix_add(&fx[og * NV1 + 1 + G + c * 256 + lane * 8 + k], (double)g[c][k]);
                            g[c][k] = 0.f;
                        }
                    double llw = ll_total + (double)ll_acc;
                    for (int o = 16; o > 0; o >>= 1) llw += __shfl_xor_sync(0xffffffffu, llw, o);
                    if (lane == 0) fed::fix_add(&fx[og * NV1], llw * 0.25);
                    ll_total = 0.0;
                    ll_acc = 0.f;
                    flush_count = 0;
                }
            }
            const long long r0 = (b - seg.first_tile) * kBatch;
            const __nv_bfloat16* Xs = reinterpret_cast<const __nv_bfloat16*>(seg.X);

            float xf[kBatch][NCH][8];
            float p[kBatch];
#pragma unroll
            for (int j = 0; j < kBatch; ++j) {
                const long long row = r0 + j;
                const bool valid = row < seg.n_rows;
                p[j] = 0.f;
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    uint4 v = make_uint4(0, 0, 0, 0);
                    if (valid && lane_on[c]) v = ldg_stream(Xs + row * (long long)prm.ld + c * 256 + lane * 8);
                    xf[j][c][0] = bf16_lo(v.x); xf[j][c][1] = bf16_hi(v.x);
                    xf[j][c][2] = bf16_lo(v.y); xf[j][c][3] = bf16_hi(v.y);
                    xf[j][c][4] = bf16_lo(v.z); xf[j][c][5] = bf16_hi(v.z);
                    xf[j][c][6] = bf16_lo(v.w); xf[j][c][7] = bf16_hi(v.w);
#pragma unroll
                    for (int k = 0; k < 8; ++k) p[j] = fmaf(xf[j][c][k], beta[c][k], p[j]);
                }
            }
            // transposing butterfly: 8 values x 32 lanes -> lane holds sum for row (lane >> 2)
            const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
            float q[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float send = b4 ? p[i] : p[i + 4];
                const float keep = b4 ? p[i + 4] : p[i];
                q[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
            float t2[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float send = b3 ? q[i] : q[i + 2];
                const float keep = b3 ? q[i + 2] : q[i];
                t2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
            float eta;
            {
                const float send = b2 ? t2[0] : t2[1];
                const float keep = b2 ? t2[1] : t2[0];
                eta = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            eta += __shfl_xor_sync(0xffffffffu, eta, 2);
            eta += __shfl_xor_sync(0xffffffffu, eta, 1);
            eta += icpt;

            const long long myrow = r0 + jrow;
            float ll = 0.f, r = 0.f;
            if (myrow < seg.n_rows) {
                const float y = __ldg(seg.y + myrow);
                // per-row offset / weight (null: absent, uniform per segment); rounded on their own, so w = 1, o = 0
                // gives the bits of the plain model, and a zero weight selects 0 over a non-finite y or offset
                if (seg.offset) eta = __fadd_rn(eta, __ldg(seg.offset + myrow));
                link_loglik(prm.family, y, eta, ll, r);
                if (seg.weight) {
                    const float wt = __ldg(seg.weight + myrow);
                    apply_weight(wt, ll);
                    apply_weight(wt, r);
                }
            }
            ll_acc += ll;
            gi += r;
#pragma unroll
            for (int j = 0; j < kBatch; ++j) {
                const float rj = __shfl_sync(0xffffffffu, r, j * 4);
#pragma unroll
                for (int c = 0; c < NCH; ++c)
#pragma unroll
                    for (int k = 0; k < 8; ++k) g[c][k] = fmaf(rj, xf[j][c][k], g[c][k]);
            }
            // keep fp32 running sums short: spill LL to fp64 every 256 batches
            if (++flush_count == 256) {
                ll_total += (double)ll_acc;
                ll_acc = 0.f;
                flush_count = 0;
            }
        }
        ll_total += (double)ll_acc;
        gi = warp_sum(gi);
        if (NOUT > 1) {
            double llw = ll_total;
            for (int o = 16; o > 0; o >>= 1) llw += __shfl_xor_sync(0xffffffffu, llw, o);
            if (b_end > gw * T / W) {
                const int og = seg.out_group;
#pragma unroll
                for (int c = 0; c < NCH; ++c)
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (lane_on[c]) fed::fix_add(&fx[og * NV1 + 1 + G + c * 256 + lane * 8 + k], (double)g[c][k]);
                if (lane == 0) {
                    fed::fix_add(&fx[og * NV1], llw * 0.25);
                    fed::fix_add(&fx[og * NV1 + 1 + seg.group], (double)gi * 0.25);
                }
            }
            __syncthreads();
            for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) out[i] = fed::fix_get(__ldcg(&fx[i]));
        } else {
        if (lane == 0 && b_end > gw * T / W) fed::fix_add(&gi_acc[seg.group], (double)gi * 0.25);

        // ---- CTA reduction -> cta_partials[blockIdx.x] = [LL, gi[G], g[P]] ----
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int k = 0; k < 8; ++k) g_red[warp * (NCH * 256) + c * 256 + lane * 8 + k] = g[c][k];
        const double ll_block = fed::block_sum(ll_total * 0.25, red);  // also syncs
        if (threadIdx.x == 0) out[0] = ll_block;
        for (int i = threadIdx.x; i < G; i += blockDim.x) out[1 + i] = fed::fix_get(gi_acc[i]);
        for (int f = threadIdx.x; f < P; f += blockDim.x) {
            double sum = 0.0;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) sum += (double)g_red[w * (NCH * 256) + f];
            out[1 + G + f] = sum;
        }
        }
    }
    fed::epilogue(comm, pro, 0ull);
}

}  // namespace

extern "C" size_t b200_glm_simt_smem(int n_theta, int n_features, int n_groups) {
    const int nch = (n_features + 255) / 256;
    return (size_t)((n_theta + 3) & ~3) * 4 + (size_t)kWarps * nch * 256 * 4 + (size_t)((n_groups + 1) & ~1) * 8 + 32 * 8;
}

extern "C" int b200_launch_glm_simt(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, int grid,
                                    cudaStream_t stream) {
    const int nch = (prm->n_features + 255) / 256;
    if (prm->n_chains != 1 || nch < 1 || nch > 2 || (prm->n_features % 8) != 0 || (prm->ld % 8) != 0) return -1;
    const size_t smem = b200_glm_simt_smem(comm->n_theta, prm->n_features, prm->n_groups);
#define LAUNCH(N)                                                                                              \
    do {                                                                                                       \
        cudaFuncSetAttribute(fed_glm_simt_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
        fed_glm_simt_kernel<N><<<grid, kWarps * 32, smem, stream>>>(*comm, segs_dev, *prm);                    \
    } while (0)
    if (nch == 1) LAUNCH(1); else LAUNCH(2);
#undef LAUNCH
    return (int)cudaGetLastError();
}
