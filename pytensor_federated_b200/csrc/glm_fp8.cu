// Federated logistic GLM on a BLOCK-SCALED FP8 design matrix (Hopper: wgmma e4m3 + TMA + mbarrier).
//
// Storage: X as e4m3 bytes + one UE8M0 scale per 32 x 32 block (32 rows x 32 features):
//     x[r, f] = e4m3(Xq[r, f]) * 2^(S[r/32, f/32] - 127)
// i.e. 1.03 bytes per element instead of 2 for bf16 -> the HBM-bound evaluation reads half the bytes.
// The scales come pre-packed per 128-row tile (models/glm.py: pack_tile_scales); this kernel reads byte
// 32 + 4 fb + q of a tile's 64 = the scale of (row group q, feature block fb).
//
// Hopper has no block-scaled MMA:
//   MMA #1  eta[64 rows x 24] = Xd_rows . Theta^T   on a dequantised bf16 copy of the consumer's rows: an e4m3
//           value times its power-of-two block scale is exact in bf16, so the copy IS the design matrix and
//           the MMA runs as one chain.  Theta is a 3-way bf16 split as in glm_tc.cu (the fp8 wgmma accumulates
//           with fewer mantissa bits than fp32, which eta, a long dot product with cancellation, cannot afford).
//   MMA #2  G[64 feat x 32] += sum_rg S[rg, fb] * s_r[rg] * (Xq^T[feat, rg] . R[rg])   in e4m3, the block scales
//           applied in fp32 registers after each 32-row K step; 8-bit wgmma operands must be K-major, so it reads
//           a transposed copy of the tile that each consumer warpgroup writes for its feature half.
// The residuals are a 4-term radix-16 e4m3 expansion (term k carries weight 16^-k) in separate N columns,
// recombined in fp32/fp64, so the low precision of the operand does not leak into the gradient.
// Poisson / Gaussian residuals are unbounded: there (template DYN) every 32-row group of R gets its own
// power-of-two scale s_r (from the group's largest |r|), so the expansion is relative to the block maximum.
// Observation weights make even logistic residuals unbounded, so weighted models take the DYN scaling too.
//
// Roles and pipeline as in glm_tc.cu.  Workload: BASELINE.json "hierarchical GLM, 8 partial-pooling groups
// (one per GPU), fp8 block-scaled design matrix" (groups = intercepts).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include "fed_comm.cuh"
#include "models.h"
#include "tc_common.cuh"
#include "chunks.h"

namespace fp8 {
using namespace tc;

constexpr int kTile = 128;            // rows per tile
constexpr int kPanelF = 128;          // features per 128-byte swizzle span (1 byte / element)
constexpr int kPanelB = kTile * 128;  // 16 KB
constexpr int kThreadsF = 384;        // warpgroup 0: TMA producer (warp 0 only), warpgroups 1, 2: consumers
constexpr int kConsumerWarpsF = 8;
constexpr int kChunkMultiple = 3;     // tiles per chunk: a multiple of this (chunk table shared with older layouts)
constexpr int kMaxChunkF = 30;        // tiles per chunk at most (fp32 register accumulation)
constexpr int kMinChunkF = 6;
constexpr int kRingF = 16;            // published chunks the consumers may lag behind
constexpr int kLLRowsF = 12;          // per-warp slot rows of the warp-level sums (>= kConsumerWarpsF)
constexpr int kResidTerms = 4;
constexpr int kN1 = 24;               // eta columns: bf16 term t (hi, mid, lo) of chain k in column 8 t + k
constexpr int kN2 = 8 * kResidTerms;  // residual columns: term t of chain k in column 8 t + k

__device__ __forceinline__ uint8_t to_e4m3(float v) {
    return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}
__device__ __forceinline__ float from_e4m3(uint8_t b) {
    const __half_raw h = __nv_cvt_fp8_to_halfraw(b, __NV_E4M3);
    return __half2float(*reinterpret_cast<const __half*>(&h));
}
// radix-16 expansion: v ~= sum_k terms[k] * 16^-k, each term an e4m3 of magnitude <= 448
template <int T>
__device__ __forceinline__ void expand16(float v, uint8_t (&terms)[T]) {
    float rem = v;
#pragma unroll
    for (int k = 0; k < T; ++k) {
        terms[k] = to_e4m3(rem);
        rem = (rem - from_e4m3(terms[k])) * 16.f;
    }
}
__device__ __forceinline__ float ue8m0(uint32_t b) { return __uint_as_float(b << 23); }

struct SmemLayoutF {
    uint32_t stages, stage_bytes, off_xb, xb_bytes, off_theta_b, theta_b_bytes, off_r, r_bytes, off_xt, xt_bytes, off_theta_f,
        off_ring, off_bars, off_misc, total;
};
// doubles per CTA row of the partial array: (hi, lo) pairs of the n_vals outputs, then the per-warp slots
// [kLLRowsF][KF][1 + G] of the warp-level sums (log-likelihood, intercept gradients) — see csrc/glm_tc.cu
__host__ __device__ constexpr size_t partial_row_doubles(int n_vals, int kf, int n_out, int n_groups) {
    return 2 * ((size_t)n_vals + (size_t)kLLRowsF * n_out * kf * (1 + n_groups));
}
__host__ __device__ inline SmemLayoutF smem_layout(int P, int n_theta, int n_groups) {
    SmemLayoutF L;
    const uint32_t panels = P / kPanelF;
    L.stage_bytes = panels * kPanelB;
    L.xb_bytes = P * 128;             // one consumer warpgroup's 64 rows in bf16: P / 64 panels of 64 rows x 128 bytes
    L.theta_b_bytes = (P / 64) * kN1 * 128;
    L.r_bytes = kTile * kN2;   // 1 byte per element
    L.xt_bytes = (P / 2) * kTile;   // one consumer warpgroup's transposed feature half
    const uint32_t fixed = 2 * L.xb_bytes + L.theta_b_bytes + 2 * L.r_bytes + 2 * L.xt_bytes + ((n_theta * 4 + 15) & ~15) +
                           kRingF * 24 + 256 + 768 + 1024;
    uint32_t stages = (227u * 1024u - fixed) / L.stage_bytes;
    if (stages > 6) stages = 6;
    L.stages = stages;
    uint32_t o = stages * L.stage_bytes;
    L.off_xb = o; o += 2 * L.xb_bytes;
    L.off_theta_b = o; o += L.theta_b_bytes;
    L.off_r = o; o += 2 * L.r_bytes;
    L.off_xt = o; o += 2 * L.xt_bytes;
    L.off_theta_f = o; o += (n_theta * 4 + 15) & ~15;
    L.off_ring = o; o += kRingF * 24;   // published chunks + one mbarrier per ring slot
    L.off_bars = o; o += 256;
    L.off_misc = o; o += 768;           // per-warp residual maxima, residual scales (DYN)
    L.total = o + 1024;
    return L;
}

// KF = chains per launch: 1 or 3; DYN = per-row-group residual scales (families with unbounded residuals, or
// weights); ROWS = some segment has per-row offsets or weights (see csrc/glm_tc.cu)
template <int KF, bool DYN, bool ROWS>
__global__ void __launch_bounds__(kThreadsF, 1)
fed_glm_fp8_kernel(FedComm comm, const GlmSegment* __restrict__ segs_g, GlmParams prm, const CUtensorMap* __restrict__ tmaps,
                   const GlmChunk* __restrict__ chunks, int n_chunks, unsigned int* __restrict__ work_counter) {
    extern __shared__ unsigned char smem_dyn[];
    // 1 KB alignment (128B-swizzled TMA tiles) by offsetting INSIDE the shared array: the pointer keeps its
    // shared address space, so the compiler emits LDS / STS instead of generic LD / ST for everything below
    unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);

    const int P = prm.n_features;
    const int G = prm.n_groups;
    const int NH = P / 128;       // 128-feature panels
    const SmemLayoutF L = smem_layout(P, comm.n_theta, G);
    const int S = (int)L.stages;

    unsigned char* theta_b = smem + L.off_theta_b;
    unsigned char* r_buf = smem + L.off_r;
    unsigned char* xt_buf = smem + L.off_xt;
    float* theta_f = reinterpret_cast<float*>(smem + L.off_theta_f);
    int4* ring = reinterpret_cast<int4*>(smem + L.off_ring);          // published chunks: (segment or -1, first tile, tiles, -)
    uint64_t* bar_ring = reinterpret_cast<uint64_t*>(smem + L.off_ring + kRingF * 16);   // slot j % kRingF: chunk j published
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    unsigned char* xb_buf = smem + L.off_xb;
    float* r_wmax = reinterpret_cast<float*>(smem + L.off_misc);            // [8 warps][8 chain slots] max |r| over 16 rows
    float* r_scale = reinterpret_cast<float*>(smem + L.off_misc + 256);     // [2 R buffers][4 row groups][8 chain slots]
    uint64_t* bar_full = bars;            // [6]
    uint64_t* bar_empty = bars + 6;       // [6]   (bars + 128 B: chunk decision)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---- theta-independent setup: BEFORE the dependency wait inside fed::prologue, so that it overlaps with the
    // tail of the previous evaluation under programmatic dependent launch (see csrc/glm_tc.cu)
    if (threadIdx.x == 0) {
        *pipeline_fault() = 0;
        for (int i = 0; i < kRingF; ++i) mbar_init(&bar_ring[i], 1);
        for (int i = 0; i < 6; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 32 * kConsumerWarpsF); }
        fence_barrier_init();
    }
    if (warp == 0 && lane == 0)
        for (int i = 0; i < prm.n_segments; ++i) tma_prefetch_desc(&tmaps[i]);
    // Early loads (see csrc/glm_tc.cu): the TMA warp claims the first chunk and fills the stage ring before
    // theta has arrived; theta has its own shared memory here, so every stage can be used.
    unsigned int claim0 = 0;
    int preloaded = 0;
    if (warp == 0) {
        __syncwarp();   // lane 0's mbarrier inits
        fed::pdl_wait();
        if (lane == 0) claim0 = atomicAdd(work_counter, 1u);
        claim0 = __shfl_sync(0xffffffffu, claim0, 0);
        if (claim0 < (unsigned int)n_chunks) {
            const GlmChunk ch = chunks[claim0];
            preloaded = ch.n_tiles < S ? ch.n_tiles : S;
            if (!prm.early_loads) preloaded = 0;
            if (elect_one()) {
                for (int t = 0; t < preloaded; ++t) {
                    mbar_expect_tx(&bar_full[t], L.stage_bytes);
                    for (int pnl = 0; pnl < NH; ++pnl)
                        tma_load_2d(smem + (size_t)t * L.stage_bytes + pnl * kPanelB, &tmaps[ch.seg], pnl * kPanelF,
                                    (ch.first_tile + t) * kTile, &bar_full[t]);
                }
            }
            __syncwarp();
        }
    }

    fed::Prologue pro = fed::prologue(comm, theta_f);   // contains __syncthreads()
    const bool active = !pro.stop && !pro.timed_out;
    constexpr float kResidNorm = 1.f / 256.f;  // r = kResidNorm * sum_k t_k 16^-k, |r| <= 1

    const int nch = prm.n_chains < KF ? prm.n_chains : KF;
    const int PG = G + P;  // parameters per chain
    const int NV1 = 1 + PG;   // outputs per chain: [LL, gi[G], g[P]]
    const int NS1 = 1 + G;    // warp-level values per chain: LL and the G intercept gradients
    // this CTA's running sums as (hi, lo) pairs (see csrc/glm_tc.cu: dynamic chunks + double-double sums)
    const int NOUT = prm.n_out;   // output blocks (1 = everything summed; else one per node, GlmSegment::out_group)
    const size_t row_doubles = partial_row_doubles(comm.n_vals, KF, NOUT, G);
    double* out = comm.cta_partials + (size_t)blockIdx.x * row_doubles;
    double* ll_slots = out + 2 * (size_t)comm.n_vals;   // [kLLRowsF][NOUT][KF][1 + G] pairs

    if (active) {
        for (size_t i = threadIdx.x; i < row_doubles / 2; i += blockDim.x) reinterpret_cast<double2*>(out)[i] = make_double2(0.0, 0.0);
        // ---- Theta^T as the K-major, 128B-swizzled bf16 B operand of MMA #1: row n = 8 * term + chain
        for (int idx = threadIdx.x; idx < (P / 64) * kN1 * 8; idx += blockDim.x) {
            const int j = idx & 7;                 // 16-byte chunk = 8 features
            const int n = (idx >> 3) % kN1;
            const int pnl = idx / (8 * kN1);
            const int chain = n % 8, term = n / 8;
            uint32_t packed[4] = {0, 0, 0, 0};
            if (chain < nch) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float v = theta_f[chain * PG + G + pnl * 64 + j * 8 + e];
                    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
                    const float rem1 = v - __bfloat162float(hi);
                    const __nv_bfloat16 mid = __float2bfloat16_rn(rem1);
                    const __nv_bfloat16 lo = __float2bfloat16_rn(rem1 - __bfloat162float(mid));
                    const __nv_bfloat16 pick = term == 0 ? hi : (term == 1 ? mid : lo);
                    packed[e >> 1] |= (uint32_t)__bfloat16_as_ushort(pick) << ((e & 1) * 16);
                }
            }
            *reinterpret_cast<uint4*>(theta_b + pnl * (kN1 * 128) + n * 128 + ((j ^ (n & 7)) * 16)) =
                make_uint4(packed[0], packed[1], packed[2], packed[3]);
        }
        fence_proxy_async();
        __syncthreads();

        // Consumers: the j-th chunk of this CTA, or x < 0 when the producer found the work counter exhausted.
        // (an mbarrier per ring slot: the producer arrives after writing the entry — release —, the consumers wait
        // on the slot's phase — acquire; slot j % kRingF is reused every kRingF chunks, consumers lag ~3 at most)
        auto next_chunk = [&](int j) -> int4 {
            mbar_wait(&bar_ring[j & (kRingF - 1)], (uint32_t)((j / kRingF) & 1));
            if (*pipeline_fault()) return make_int4(-1, 0, 0, 0);   // a stalled pipeline ends every role loop
            return ring[j & (kRingF - 1)];
        };
        // Consumers decide each chunk together: both warpgroups meet at named barriers, so one of them leaving on
        // a stalled pipeline while the other waits at a barrier would hang.  One thread reads the fault flag and
        // the ring entry after all 256 have arrived and shares the decision through shared memory.
        int4* chunk_decided = reinterpret_cast<int4*>(smem + L.off_bars + 128);
        auto consumer_chunk = [&](int j) -> int4 {
            const int slot = j & (kRingF - 1);
            mbar_wait(&bar_ring[slot], (uint32_t)((j / kRingF) & 1));
            named_sync(1, 256);
            if (threadIdx.x == 128) *chunk_decided = *pipeline_fault() ? make_int4(-1, 0, 0, 0) : ring[slot];
            named_sync(1, 256);
            return *chunk_decided;
        };

        if (warp == 0) {
            // ================= TMA producer + chunk scheduler (see csrc/glm_tc.cu) ==============
            Ring stage;
            unsigned int claim = claim0, ahead = 0;   // the first chunk was claimed before theta arrived
            for (int j = 0;; ++j) {
                const bool have = claim < (unsigned int)n_chunks;
                GlmChunk ch{};
                if (have) ch = chunks[claim];
                if (lane == 0) {
                    ring[j & (kRingF - 1)] = have ? make_int4(ch.seg, ch.first_tile, ch.n_tiles, 0) : make_int4(-1, 0, 0, 0);
                    mbar_arrive(&bar_ring[j & (kRingF - 1)]);
                    if (have) ahead = atomicAdd(work_counter, 1u);
                }
                __syncwarp();
                if (!have) break;
                for (int t = 0; t < ch.n_tiles; ++t) {
                    const int st = stage.idx;
                    if (j == 0 && t < preloaded) {   // already in flight (early loads)
                        stage.advance(S);
                        continue;
                    }
                    mbar_wait(&bar_empty[st], stage.phase ^ 1);
                    const int row0 = (ch.first_tile + t) * kTile;
                    unsigned char* dst = smem + (size_t)st * L.stage_bytes;
                    if (elect_one()) {
                        mbar_expect_tx(&bar_full[st], L.stage_bytes);
                        for (int pnl = 0; pnl < NH; ++pnl)
                            tma_load_2d(dst + pnl * kPanelB, &tmaps[ch.seg], pnl * kPanelF, row0, &bar_full[st]);
                    }
                    __syncwarp();
                    stage.advance(S);
                }
                claim = __shfl_sync(0xffffffffu, ahead, 0);
            }
        } else if (warp >= 4) {
            // ================= consumer warpgroups: rows 64c .. 64c + 63 (eta), features c P/2 .. (gradient)
            const int c = (warp >> 2) - 1;
            const int w = warp & 3;
            const int q = lane & 3;
            const int ew = warp - 4;                 // consumer warp ordinal: row of the per-warp slots
            const int tid = threadIdx.x - 128 * (c + 1);
            const int rg_me = 2 * c + (w >> 1);     // row group of this thread's two eta rows
            const int NB = P / 128;                  // 64-feature gradient blocks per warpgroup (1 or 2)
            const uint64_t desc_x = make_desc(0, 16, 1024, 1);      // bf16 X rows / Theta^T: K-major, 128B swizzle
            const uint64_t desc_kn = make_desc(0, 128, 1024, 0);    // X^T copy and R: K-major, no swizzle
            const uint32_t theta_b_a = smem_u32(theta_b);
            const uint32_t x_base_a = smem_u32(smem);
            const uint32_t r_a = smem_u32(r_buf);
            unsigned char* xt = xt_buf + c * L.xt_bytes;
            const uint32_t xt_a = smem_u32(xt);
            unsigned char* xb = xb_buf + c * L.xb_bytes;
            const uint32_t xb_a = smem_u32(xb);
            float gacc[2][kN2 / 2];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int v = 0; v < kN2 / 2; ++v) gacc[i][v] = 0.f;
            Ring stage;
            uint32_t rb = 0;   // R buffer of the current tile (alternates)
            for (int j = 0;; ++j) {
                const int4 ch = consumer_chunk(j);
                if (ch.x < 0) break;
                const float* __restrict__ seg_y = segs_g[ch.x].y;
                const float* __restrict__ seg_o = ROWS ? segs_g[ch.x].offset : nullptr;   // null: absent (chunk-uniform)
                const float* __restrict__ seg_w = ROWS ? segs_g[ch.x].weight : nullptr;
                const long long seg_rows = segs_g[ch.x].n_rows;
                const long long seg_tiles = (seg_rows + kTile - 1) / kTile;
                const uint8_t* __restrict__ seg_sc = reinterpret_cast<const uint8_t*>(segs_g[ch.x].scales);
                const int seg_group = segs_g[ch.x].group;
                const int og = segs_g[ch.x].out_group;   // output block of this chunk's segment
                float ll_acc[2], gi_acc[2];
                ll_acc[0] = ll_acc[1] = gi_acc[0] = gi_acc[1] = 0.f;
                for (int t = 0; t < ch.z; ++t) {
                    // block scales of this tile (an empty tile that pads a chunk: 2^0, its rows are zero)
                    const long long tile = (long long)ch.y + t;
                    const uint8_t* sc = seg_sc + (size_t)tile * 64 + 32;   // byte 4 fb + rg
                    const bool real_tile = tile < seg_tiles;
                    float s2[4][2];
#pragma unroll
                    for (int rg = 0; rg < 4; ++rg)
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int fb = c * (P / 64) + 2 * i + (w >> 1);
                            s2[rg][i] = (real_tile && i < NB) ? ue8m0(__ldg(sc + 4 * fb + rg)) : 1.f;
                        }
                    mbar_wait(&bar_full[stage.idx], stage.phase);
                    const uint32_t x_a = x_base_a + (uint32_t)stage.idx * L.stage_bytes;
                    const unsigned char* xs = smem + (size_t)stage.idx * L.stage_bytes;
                    // ---- dequantised bf16 copy of this group's 64 rows (64-feature panels of 64 rows x 128 bytes, 128B
                    // swizzle): an e4m3 value times its power-of-two block scale is exact in bf16
                    for (int b = tid; b < 64 * (P / 16); b += 128) {
                        const int r = b / (P / 16);              // row within the group
                        const int f = (b % (P / 16)) * 16;       // first of 16 features (one scale block)
                        const int rr = 64 * c + r, fi = f & 127;
                        const float bs = real_tile ? ue8m0(__ldg(sc + 4 * (f >> 5) + (rr >> 5))) : 1.f;
                        const uint4 v = *reinterpret_cast<const uint4*>(xs + (f >> 7) * kPanelB + rr * 128 + (((fi >> 4) ^ (rr & 7)) << 4));
                        const uint32_t wds[4] = {v.x, v.y, v.z, v.w};
                        uint32_t o[8];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(wds[i] & 0xFFFFu), __NV_E4M3);
                            const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(wds[i] >> 16), __NV_E4M3);
                            const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&lo));
                            const float2 a1 = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                            const __nv_bfloat162 b0 = __floats2bfloat162_rn(a0.x * bs, a0.y * bs), b1 = __floats2bfloat162_rn(a1.x * bs, a1.y * bs);
                            o[2 * i] = *reinterpret_cast<const uint32_t*>(&b0);
                            o[2 * i + 1] = *reinterpret_cast<const uint32_t*>(&b1);
                        }
                        const int jb = (f & 63) >> 3;            // first of the two 8-feature chunks in the bf16 panel
                        unsigned char* dst = xb + (f >> 6) * 8192 + r * 128;
                        *reinterpret_cast<uint4*>(dst + ((jb ^ (r & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
                        *reinterpret_cast<uint4*>(dst + (((jb + 1) ^ (r & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
                    }
                    fence_proxy_async();
                    named_sync(2 + c, 128);
                    // ---- MMA #1 on the dequantised rows: one uninterrupted chain of K steps
                    float eacc[kN1 / 2];
#pragma unroll
                    for (int v = 0; v < kN1 / 2; ++v) eacc[v] = 0.f;
                    wgmma_fence();
                    for (int pnl = 0; pnl < P / 64; ++pnl) {
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks)
                            wgmma_bf16<kN1, 0, 0>(eacc, desc_x | (uint64_t)((xb_a + pnl * 8192 + ks * 32) >> 4),
                                                  desc_x | (uint64_t)((theta_b_a + pnl * (kN1 * 128) + ks * 32) >> 4), (pnl | ks) ? 1u : 0u);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(eacc);
                    // ---- transposed copy of this group's feature half: element (feature fl, row r) at
                    // (fl / 8) * 1024 + (r / 16) * 128 + (fl % 8) * 16 + r % 16; 4 x 4 byte blocks through registers
                    for (int b = tid; b < (P / 8) * (kTile / 4); b += 128) {
                        const int fl = (b % (P / 8)) * 4;        // first of 4 features (local to the half)
                        const int r = (b / (P / 8)) * 4;         // first of 4 rows
                        const int f = c * (P / 2) + fl;
                        const int fi = f & 127;
                        uint32_t a[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int rr = r + i;
                            a[i] = *reinterpret_cast<const uint32_t*>(xs + (f >> 7) * kPanelB + rr * 128 +
                                                                      ((((fi >> 4) ^ (rr & 7))) << 4) + (fi & 15));
                        }
                        const uint32_t t0 = __byte_perm(a[0], a[1], 0x5140), t1 = __byte_perm(a[2], a[3], 0x5140);
                        const uint32_t t2 = __byte_perm(a[0], a[1], 0x7362), t3 = __byte_perm(a[2], a[3], 0x7362);
                        const uint32_t o[4] = {__byte_perm(t0, t1, 0x5410), __byte_perm(t0, t1, 0x7632),
                                               __byte_perm(t2, t3, 0x5410), __byte_perm(t2, t3, 0x7632)};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int fr = fl + i;
                            *reinterpret_cast<uint32_t*>(xt + (fr >> 3) * 1024 + (r >> 4) * 128 + (fr & 7) * 16 + (r & 15)) = o[i];
                        }
                    }
                    // ---- link, likelihood, residual -> 4 e4m3 terms per chain in R (element (row, n) at
                    // (n / 8) * 1024 + (row / 16) * 128 + (n % 8) * 16 + row % 16)
                    float rr_[2][2];
                    float yv[2];
                    bool valid[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = 64 * c + 16 * w + (lane >> 2) + 8 * h;
                        const long long grow = tile * kTile + row;
                        valid[h] = grow < seg_rows;
                        yv[h] = valid[h] ? __ldg(seg_y + grow) : 0.f;
                        float o = 0.f, wt = 1.f;   // offset and weight of the row
                        if constexpr (ROWS) {
                            if (valid[h] && seg_o) o = __ldg(seg_o + grow);
                            if (valid[h] && seg_w) wt = __ldg(seg_w + grow);
                        }
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int k = 2 * q + e;
                            const int kk = k < KF ? k : 0;
                            float eta = (eacc[2 * h + e] + eacc[4 + 2 * h + e]) + eacc[8 + 2 * h + e] + theta_f[kk * PG + seg_group];
                            if constexpr (ROWS) eta = __fadd_rn(eta, o);   // offset after the intercept
                            float ll = 0.f, r = 0.f;
                            if (valid[h] && k < nch) {
                                link_loglik(DYN ? prm.family : 0, yv[h], eta, ll, r);
                                if constexpr (ROWS) {   // weight after the likelihood; a zero weight selects 0
                                    ll = wt == 0.f ? 0.f : __fmul_rn(wt, ll);
                                    r = wt == 0.f ? 0.f : __fmul_rn(wt, r);
                                }
                            }
                            ll_acc[e] += ll;
                            gi_acc[e] += r;
                            rr_[h][e] = r;
                        }
                    }
                    float rsc[2] = {1.f, 1.f};   // DYN: 2^e of this row group, max|r| / 2^e in [0.5, 1)
                    if constexpr (DYN) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float m = fmaxf(fabsf(rr_[0][e]), fabsf(rr_[1][e]));
#pragma unroll
                            for (int o = 4; o < 32; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                            if (lane < 4) r_wmax[ew * 8 + 2 * q + e] = m;
                        }
                        named_sync(2 + c, 128);
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float m = fmaxf(r_wmax[(ew & ~1) * 8 + 2 * q + e], r_wmax[(ew | 1) * 8 + 2 * q + e]);
                            int ex = 0;
                            if (m > 0.f) frexpf(m, &ex);
                            ex = max(-126, min(126, ex));
                            rsc[e] = __uint_as_float((uint32_t)(127 + ex) << 23);
                            if ((w & 1) == 0 && lane < 4) r_scale[(rb * 4 + rg_me) * 8 + 2 * q + e] = rsc[e];
                        }
                    }
                    unsigned char* rbuf = r_buf + rb * L.r_bytes;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = 64 * c + 16 * w + (lane >> 2) + 8 * h;
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            uint8_t rt[kResidTerms];
                            expand16<kResidTerms>(rr_[h][e] / rsc[e] * 256.f, rt);
#pragma unroll
                            for (int tt = 0; tt < kResidTerms; ++tt)
                                rbuf[tt * 1024 + (row >> 4) * 128 + (2 * q + e) * 16 + (row & 15)] = rt[tt];
                        }
                    }
                    fence_proxy_async();
                    named_sync(1, 32 * kConsumerWarpsF);   // R (and the residual scales) of all 128 rows written
                    // ---- MMA #2, one 32-row group per K step, scaled in registers
#pragma unroll
                    for (int rg = 0; rg < 4; ++rg) {
                        float tmp[2][kN2 / 2];
#pragma unroll
                        for (int i = 0; i < 2; ++i)
#pragma unroll
                            for (int v = 0; v < kN2 / 2; ++v) tmp[i][v] = 0.f;
                        wgmma_fence();
#pragma unroll
                        for (int i = 0; i < 2; ++i)
                            if (i < NB)
                                wgmma_e4m3<kN2>(tmp[i], desc_kn | (uint64_t)((xt_a + i * 8 * 1024 + rg * 256) >> 4),
                                                desc_kn | (uint64_t)((r_a + rb * L.r_bytes + rg * 256) >> 4), 0u);
                        wgmma_commit();
                        wgmma_wait<0>();
                        float srg[2] = {1.f, 1.f};
                        if constexpr (DYN) {
                            srg[0] = r_scale[(rb * 4 + rg) * 8 + 2 * q];
                            srg[1] = r_scale[(rb * 4 + rg) * 8 + 2 * q + 1];
                        }
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            fence_regs(tmp[i]);
                            if (i < NB)
#pragma unroll
                                for (int v = 0; v < kN2 / 2; ++v) gacc[i][v] = fmaf(s2[rg][i] * srg[v & 1], tmp[i][v], gacc[i][v]);
                        }
                    }
                    mbar_arrive(&bar_empty[stage.idx]);   // this thread is done with the X stage
                    stage.advance(S);
                    rb ^= 1u;
                }
                // ---- end of the chunk: per-thread fp32 sums -> fixed butterfly over the 8 lanes that share the
                // chains (double) -> lanes 0..3 add the warp's value to its own (hi, lo) slot; all chunk-determined
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    double lsum = (double)ll_acc[e], gsum = (double)gi_acc[e];
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
                        gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
                    }
                    const int k = 2 * q + e;
                    if (lane < 4 && k < nch) {
                        double* slot = ll_slots + 2 * ((((size_t)ew * NOUT + og) * KF + k) * NS1);
                        dd_accumulate(slot, lsum);
                        dd_accumulate(slot + 2 * (1 + seg_group), gsum);
                    }
                }
                // gradient: feature f = c P/2 + 64 i + 16 w + lane / 4 + 8 h, chain k = 2q + e, terms in columns 8 t + k
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (i < NB) {
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int f = c * (P / 2) + 64 * i + 16 * w + (lane >> 2) + 8 * h;
                                const int k = 2 * q + e;
                                if (k < nch)
                                    dd_accumulate(out + 2 * (((size_t)og * nch + k) * NV1 + 1 + G + f),
                                                  (double)kResidNorm * ((double)gacc[i][2 * h + e] + (double)gacc[i][4 + 2 * h + e] * (1.0 / 16) +
                                                                        (double)gacc[i][8 + 2 * h + e] * (1.0 / 256) +
                                                                        (double)gacc[i][12 + 2 * h + e] * (1.0 / 4096)));
                            }
                    }
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int v = 0; v < kN2 / 2; ++v) gacc[i][v] = 0.f;
            }
        }

        __syncthreads();
        fed::pdl_trigger();   // the next evaluation's CTA may take this SM as soon as we exit
        // layout per chain: [LL, gi[G], g[P]] as (hi, lo) pairs; g[] was accumulated in place, LL and gi[] are the
        // per-warp slots summed in warp order
        for (int i = threadIdx.x; i < NOUT * nch * NS1; i += blockDim.x) {
            const int jv = i % NS1, k = (i / NS1) % nch, o = i / (NS1 * nch);
            double hi = 0.0, lo = 0.0;
            for (int w = 0; w < kConsumerWarpsF; ++w) {
                const double* slot = ll_slots + 2 * ((((size_t)w * NOUT + o) * KF + k) * NS1 + jv);
                fed::dd_add(hi, lo, slot[0], slot[1]);
            }
            out[2 * (((size_t)o * nch + k) * NV1 + jv)] = hi;
            out[2 * (((size_t)o * nch + k) * NV1 + jv) + 1] = lo;
        }
    } else if (warp == 0) {
        // nothing will be computed (stop / idle): the early loads still have to land before the CTA may exit
        for (int t = 0; t < preloaded; ++t) mbar_wait(&bar_full[t], 0u);
    }
    __syncthreads();
    const bool fin = fed::epilogue_t<true>(comm, pro, (active && *pipeline_fault()) ? B200FED_ERR_PIPELINE : 0ull, row_doubles,
                                           comm.group_partials);
    if (fin && threadIdx.x == 0) *work_counter = 0u;   // every CTA has stopped claiming: ready for the next launch
}

}  // namespace fp8

extern "C" int b200_glm_fp8_prepare(const GlmSegment* segs_host, int n_segments, const GlmParams* prm, int sm_count,
                                    void** tmaps_dev, void** chunks_dev, int* n_chunks) {
    if (prm->n_features != 128 && prm->n_features != 256) return -21;   // <= 8 scale blocks per tile row
    for (int s = 0; s < n_segments; ++s)
        if (segs_host[s].n_rows + fp8::kTile * fp8::kChunkMultiple >= (1ll << 31)) return -22;   // row coordinates are 32-bit
    if (prm->n_chains < 1 || prm->n_chains > 3 || prm->family < 0 || prm->family > 2) return -23;
    if (prm->ld % 16 != 0) return -24;
    const PFN_cuTensorMapEncodeTiled encode = tc::encode_tiled();
    if (!encode) return -25;
    CUtensorMap* host = new CUtensorMap[n_segments];
    for (int s = 0; s < n_segments; ++s) {
        if (((uintptr_t)segs_host[s].X & 15) != 0 || segs_host[s].scales == nullptr) { delete[] host; return -26; }
        cuuint64_t dims[2] = {(cuuint64_t)prm->n_features, (cuuint64_t)segs_host[s].n_rows};
        cuuint64_t strides[1] = {(cuuint64_t)prm->ld};
        cuuint32_t box[2] = {(cuuint32_t)fp8::kPanelF, (cuuint32_t)fp8::kTile};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&host[s], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(segs_host[s].X), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { delete[] host; return -27; }
    }
    if (*tmaps_dev) cudaFree(*tmaps_dev);
    cudaError_t e = cudaMalloc(tmaps_dev, sizeof(CUtensorMap) * n_segments);
    if (e == cudaSuccess) e = cudaMemcpy(*tmaps_dev, host, sizeof(CUtensorMap) * n_segments, cudaMemcpyHostToDevice);
    delete[] host;
    if (e != cudaSuccess) return (int)e;
    const std::vector<GlmChunk> chunks = build_chunks(segs_host, n_segments, sm_count > 0 ? sm_count : 132, fp8::kTile, fp8::kChunkMultiple,
                                                        fp8::kMaxChunkF, fp8::kMinChunkF);
    if (*chunks_dev) cudaFree(*chunks_dev);
    e = cudaMalloc(chunks_dev, sizeof(GlmChunk) * (chunks.size() + 1));
    if (e == cudaSuccess) e = cudaMemcpy(*chunks_dev, chunks.data(), sizeof(GlmChunk) * chunks.size(), cudaMemcpyHostToDevice);
    *n_chunks = (int)chunks.size();
    return e == cudaSuccess ? 0 : (int)e;
}

extern "C" size_t b200_glm_fp8_partial_row_doubles(int n_vals, int n_chains, int n_out, int n_groups) {
    return fp8::partial_row_doubles(n_vals, n_chains == 1 ? 1 : 3, n_out > 0 ? n_out : 1, n_groups);
}

extern "C" int b200_launch_glm_fp8(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, const void* tmaps,
                                   const void* chunks_dev, int n_chunks, unsigned int* work_counter, int grid,
                                   cudaStream_t stream) {
    const fp8::SmemLayoutF L = fp8::smem_layout(prm->n_features, comm->n_theta, prm->n_groups);
    if (L.stages < 2) return -2;
    // unbounded residuals (Poisson, Gaussian, or any weighted model): per-row-group scales for the R operand
    const bool dyn = prm->family != 0 || (prm->row_data & kGlmRowWeights);
    const bool rows = prm->row_data != 0;
    using fp8::fed_glm_fp8_kernel;
    const auto kernel = prm->n_chains == 1
        ? (rows ? (dyn ? fed_glm_fp8_kernel<1, true, true> : fed_glm_fp8_kernel<1, false, true>)
                : (dyn ? fed_glm_fp8_kernel<1, true, false> : fed_glm_fp8_kernel<1, false, false>))
        : (rows ? (dyn ? fed_glm_fp8_kernel<3, true, true> : fed_glm_fp8_kernel<3, false, true>)
                : (dyn ? fed_glm_fp8_kernel<3, true, false> : fed_glm_fp8_kernel<3, false, false>));
    return tc::launch_pdl(kernel, grid, fp8::kThreadsF, L.total, stream, *comm, segs_dev, *prm,
                          reinterpret_cast<const CUtensorMap*>(tmaps), reinterpret_cast<const GlmChunk*>(chunks_dev),
                          n_chunks, work_counter);
}
