// Federated GLM log-likelihood + gradient on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Per 128-row tile of the bf16 design matrix X (read from HBM exactly ONCE per evaluation):
//
//   TMA        X[128 x P] -> smem, 128B-swizzled 64-feature panels (cp.async.bulk.tensor)
//   MMA #1     eta[128 x N1] = X_tile (A, K-major) . Theta^T (B, K-major)      -> registers
//              Theta holds, per MCMC chain, a 3-way bf16 split (hi, mid, lo) of the fp32
//              coefficients, so eta keeps ~fp32 accuracy although the operands are bf16.
//   epilogue   link + log-likelihood; residual r = dll/deta;
//              r is split into (hi, lo) bf16 and stored to smem as the B operand of MMA #2
//   MMA #2     G[P x N2] += X_tile^T (A, **MN-major view of the very same smem tile**) . R
//              accumulated in registers over the tiles of a chunk, then added to fp64 pairs
//
// so the gradient GEMM costs no second pass over X.  Chains are batched along N (the MMA is
// otherwise idle: the kernel is HBM-bound), which is what makes tensor cores pay here.
// Roles: warp 0 = TMA producer; consumer warpgroups 1 and 2 (warps 4-11) share every tile: warpgroup c
// computes eta / the residuals of rows 64c .. 64c + 63 and the gradient of features c P/2 .. (c + 1) P/2 - 1,
// so every gradient value has one owner thread.  One 256-thread barrier per tile publishes R; the two R
// buffers alternate, so a buffer is rewritten only after both warpgroups have passed the next tile's barrier.
// The federation prologue/epilogue (theta broadcast, NVLink reduce) is fed_comm.cuh.
//
// Workload: BASELINE.json "federated logistic GLM, 10M rows x 256 features per shard, bf16".
#include <vector>

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "fed_comm.cuh"
#include "models.h"
#include "tc_common.cuh"
#include "chunks.h"

namespace tc {

constexpr int kTileM = 128;          // rows per tile
constexpr int kPanel = 64;           // features per 128-byte swizzle span
constexpr int kPanelBytes = kTileM * 128;  // 16 KB
constexpr int kThreads = 384;        // warpgroup 0: TMA producer (warp 0 only), warpgroups 1, 2: consumers
constexpr int kConsumerWarps = 8;
constexpr int kMaxChunk = 32;        // tiles per chunk at most (= tiles accumulated in fp32 registers before a flush)
constexpr int kMinChunk = 4;
constexpr int kRing = 16;            // published chunks the consumers may lag behind (needs only ~3)
constexpr int kLLRows = 16;          // per-warp log-likelihood slot rows (>= kConsumerWarps)

struct SmemLayout {
    uint32_t stages, stage_bytes, off_theta_b, theta_b_bytes, off_r, r_bytes, off_theta_f, off_icpt, off_ring,
        off_bars, total, preload;
};
__host__ __device__ inline SmemLayout smem_layout(int P, int n1, int n2, int n_theta, int n_groups, int chains) {
    SmemLayout L;
    const uint32_t panels = P / kPanel;
    L.stage_bytes = panels * kPanelBytes;
    L.theta_b_bytes = panels * n1 * 128;
    L.r_bytes = kTileM * n2 * 2;
    // theta (fp32) is staged inside the TMA stage ring and is dead once the bf16 B operand and the intercept
    // table are built, so it costs no shared memory of its own.
    const uint32_t fixed = L.theta_b_bytes + 2 * L.r_bytes + ((chains * n_groups * 4 + 15) & ~15) + kRing * 24 + 192 +
                           1024 /*alignment slack*/;
    uint32_t stages = (227u * 1024u - fixed) / L.stage_bytes;
    if (stages > 4) stages = 4;
    L.stages = stages;
    uint32_t o = stages * L.stage_bytes;
    L.off_theta_b = o; o += L.theta_b_bytes;
    L.off_r = o; o += 2 * L.r_bytes;
    // theta (fp32) sits in the LAST stage when it fits into one: the TMA warp fills the first stages - 1 stages
    // with this CTA's first tiles BEFORE theta has arrived (`preload`), the last stage is free once the B
    // operand is built.  (larger theta: stage 0 onwards, needs n_theta * 4 <= stages * stage_bytes, no preload)
    const bool theta_in_last = (uint32_t)n_theta * 4u <= L.stage_bytes && stages >= 2;
    L.off_theta_f = theta_in_last ? (stages - 1) * L.stage_bytes : 0;
    L.preload = theta_in_last ? stages - 1 : 0;
    L.off_icpt = o; o += (chains * n_groups * 4 + 15) & ~15;
    L.off_ring = o; o += kRing * 24;   // published chunks + one mbarrier per ring slot
    L.off_bars = o; o += 192;
    L.total = o + 1024;
    return L;
}

// KC = chains per launch.  Column layouts follow the wgmma accumulator fragment (thread lane owns columns
// 8j + 2 (lane % 4) + {0, 1}), so that one thread holds every term of the chains it works on.
template <int KC>
struct Cfg {
    static constexpr int C8 = KC <= 8 ? 8 : 16;           // chain columns per theta term
    static constexpr int N1 = 3 * C8;                     // eta: term t of chain k in column t * C8 + k
    static constexpr int N2 = ((2 * KC + 7) / 8) * 8;     // residual: (hi, lo) of chain k in columns 2k, 2k + 1
};

// doubles per CTA row of the partial array: (hi, lo) pairs of the n_vals outputs, then the per-warp slots of
// the values that a whole warp contributes to — [kLLRows][n_out][KC][1 + G]: log-likelihood and the G
// intercept gradients of every (output block, chain)
__host__ __device__ constexpr size_t partial_row_doubles(int n_vals, int kc, int n_out, int n_groups) {
    return 2 * ((size_t)n_vals + (size_t)kLLRows * n_out * kc * (1 + n_groups));
}

// Work is handed out in CHUNKS of consecutive tiles of one segment (host-built table: 32 tiles while much
// work is left, shrinking to 4 towards the end; always an even number, a segment with an odd tile count
// gets one empty tile).  The TMA warp claims chunks from a global counter and publishes them to the other
// roles through a small shared-memory ring, so CTAs on faster SMs simply take more chunks: no CTA waits on
// a statically assigned straggler.  Everything a chunk contributes (fp32 register accumulation over its tiles,
// per-thread fp32 sums) depends on the chunk alone, and chunk results are combined as double-double pairs
// (fed::dd_add), so the evaluation stays reproducible although the assignment is not.
template <int KC>
__global__ void __launch_bounds__(kThreads, 1)
fed_glm_tc_kernel(FedComm comm, const GlmSegment* __restrict__ segs_g, GlmParams prm, const CUtensorMap* __restrict__ tmaps,
                  const GlmChunk* __restrict__ chunks, int n_chunks, unsigned int* __restrict__ work_counter) {
    constexpr int C8 = Cfg<KC>::C8;
    constexpr int N1 = Cfg<KC>::N1;
    constexpr int N2 = Cfg<KC>::N2;
    extern __shared__ unsigned char smem_dyn[];
    // 1 KB alignment (128B-swizzled TMA tiles) by offsetting INSIDE the shared array: the pointer keeps its
    // shared address space, so the compiler emits LDS / STS instead of generic LD / ST for everything below
    unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);

    const int P = prm.n_features;     // real number of features (theta / result layout)
    const int PP = (P + 127) & ~127;  // features the tile is padded to: TMA zero-fills the columns past P, their
                                      // Theta rows are zero and their gradient rows are never stored
    const int G = prm.n_groups;
    const int panels = PP / kPanel;
    const SmemLayout L = smem_layout(PP, N1, N2, comm.n_theta, G, KC);
    const int S = (int)L.stages;
    const int nch = prm.n_chains < KC ? prm.n_chains : KC;  // chains actually present in theta
    const int NV1 = 1 + G + P;        // outputs per chain: [LL, gi[G], g[P]]

    unsigned char* theta_b = smem + L.off_theta_b;
    unsigned char* r_buf = smem + L.off_r;
    float* theta_f = reinterpret_cast<float*>(smem + L.off_theta_f);  // valid until the setup barrier only
    float* icpt = reinterpret_cast<float*>(smem + L.off_icpt);        // [KC][G] intercepts
    int4* ring = reinterpret_cast<int4*>(smem + L.off_ring);          // (segment or -1, first row, tiles, -)
    uint64_t* bar_ring = reinterpret_cast<uint64_t*>(smem + L.off_ring + kRing * 16);   // slot j % kRing: chunk j published
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    uint64_t* bar_full = bars;            // [4] X stage landed
    uint64_t* bar_empty = bars + 4;       // [4] X stage consumed by both consumer warpgroups (bars + 128 B: chunk decision)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---------------- theta-independent setup: runs BEFORE the dependency wait inside fed::prologue, i.e. it
    // overlaps with the tail of the previous evaluation when launched with programmatic stream serialization
    if (threadIdx.x == 0) {
        *pipeline_fault() = 0;
        for (int i = 0; i < kRing; ++i) mbar_init(&bar_ring[i], 1);
        for (int i = 0; i < 4; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 32 * kConsumerWarps); }
        fence_barrier_init();
    }
    if (warp == 0 && lane == 0)
        for (int i = 0; i < prm.n_segments; ++i) tma_prefetch_desc(&tmaps[i]);
    // Early loads: X does not depend on theta.  The TMA warp waits for the previous evaluation to retire (its
    // last CTA re-arms the work counter), claims this CTA's first chunk and fills all stages but the one theta
    // is staged in, so the tensor core has `preload` tiles waiting when theta arrives (peers see theta several
    // microseconds after they became resident: root's PCIe read + the NVLink broadcast).
    unsigned int claim0 = 0;
    int preloaded = 0;
    if (warp == 0) {
        __syncwarp();   // lane 0's mbarrier inits
        fed::pdl_wait();
        if (lane == 0) claim0 = atomicAdd(work_counter, 1u);
        claim0 = __shfl_sync(0xffffffffu, claim0, 0);
        if (claim0 < (unsigned int)n_chunks) {
            const GlmChunk ch = chunks[claim0];
            preloaded = ch.n_tiles < (int)L.preload ? ch.n_tiles : (int)L.preload;
            if (!prm.early_loads) preloaded = 0;
            if (elect_one()) {
                for (int t = 0; t < preloaded; ++t) {
                    mbar_expect_tx(&bar_full[t], L.stage_bytes);
                    for (int pnl = 0; pnl < panels; ++pnl)
                        tma_load_2d(smem + (size_t)t * L.stage_bytes + pnl * kPanelBytes, &tmaps[ch.seg], pnl * kPanel,
                                    (ch.first_tile + t) * kTileM, &bar_full[t]);
                }
            }
            __syncwarp();
        }
    }

    fed::Prologue pro = fed::prologue(comm, theta_f);   // contains __syncthreads()
    const bool active = !pro.stop && !pro.timed_out;
    const int NOUT = prm.n_out;       // output blocks (1 = everything summed; else one per node)
    const int NS1 = 1 + G;            // warp-level values per (block, chain): LL and the G intercept gradients
    const size_t row_doubles = partial_row_doubles(comm.n_vals, KC, NOUT, G);
    double* out = comm.cta_partials + (size_t)blockIdx.x * row_doubles;   // this CTA's running sums, (hi, lo) pairs
    double* ll_slots = out + 2 * (size_t)comm.n_vals;                     // [kLLRows][NOUT][KC][1 + G] pairs

    if (active) {
        // ---------------- theta-dependent setup --------------------------------------------------
        for (size_t i = threadIdx.x; i < row_doubles / 2; i += blockDim.x) reinterpret_cast<double2*>(out)[i] = make_double2(0.0, 0.0);
        for (int i = threadIdx.x; i < KC * G; i += blockDim.x)
            icpt[i] = (i / G) < nch ? theta_f[(i / G) * (G + P) + (i % G)] : 0.f;
        // Theta^T as the K-major, 128B-swizzled B operand of MMA #1: row n = term * C8 + chain
        for (int idx = threadIdx.x; idx < panels * N1 * 8; idx += blockDim.x) {
            const int j = idx & 7;              // 16-byte chunk (8 features) within the 128-byte row
            const int n = (idx >> 3) % N1;
            const int pnl = idx / (8 * N1);
            const int chain = n % C8, term = n / C8;
            uint32_t packed[4] = {0, 0, 0, 0};
            if (chain < nch) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int f = pnl * kPanel + j * 8 + e;
                    const float v = f < P ? theta_f[chain * (G + P) + G + f] : 0.f;
                    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
                    const float rem1 = v - __bfloat162float(hi);
                    const __nv_bfloat16 mid = __float2bfloat16_rn(rem1);
                    const __nv_bfloat16 lo = __float2bfloat16_rn(rem1 - __bfloat162float(mid));
                    const __nv_bfloat16 pick = term == 0 ? hi : (term == 1 ? mid : lo);
                    const uint32_t bits = (uint32_t)__bfloat16_as_ushort(pick);
                    packed[e >> 1] |= bits << ((e & 1) * 16);
                }
            }
            uint4* dst = reinterpret_cast<uint4*>(theta_b + pnl * (N1 * 128) + n * 128 + ((j ^ (n & 7)) * 16));
            *dst = make_uint4(packed[0], packed[1], packed[2], packed[3]);
        }
        fence_proxy_async();
        __syncthreads();
        if (threadIdx.x == 0) fed::stamp(comm, 2);

        // Consumers: the j-th chunk of this CTA, or x < 0 when the producer found the work counter exhausted.
        // (an mbarrier per ring slot: the producer arrives after writing the entry — release —, the consumers wait
        // on the slot's phase — acquire; slot j % kRing is reused every kRing chunks, consumers lag ~3 at most)
        auto next_chunk = [&](int j) -> int4 {
            mbar_wait(&bar_ring[j & (kRing - 1)], (uint32_t)((j / kRing) & 1));
            if (*pipeline_fault()) return make_int4(-1, 0, 0, 0);   // a stalled pipeline ends every role loop
            return ring[j & (kRing - 1)];
        };
        // Consumers decide each chunk together: both warpgroups meet at named barriers, so one of them leaving on
        // a stalled pipeline while the other waits at a barrier would hang.  One thread reads the fault flag and
        // the ring entry after all 256 have arrived and shares the decision through shared memory.
        int4* chunk_decided = reinterpret_cast<int4*>(smem + L.off_bars + 128);
        auto consumer_chunk = [&](int j) -> int4 {
            const int slot = j & (kRing - 1);
            mbar_wait(&bar_ring[slot], (uint32_t)((j / kRing) & 1));
            named_sync(1, 256);
            if (threadIdx.x == 128) *chunk_decided = *pipeline_fault() ? make_int4(-1, 0, 0, 0) : ring[slot];
            named_sync(1, 256);
            return *chunk_decided;
        };

        if (warp == 0) {
            // ================= TMA producer + chunk scheduler ==================================
            // The role loops are warp-uniform (all 32 lanes wait and count); only the issue is predicated on
            // elect.sync, so the compiler keeps addresses / descriptors in uniform registers.
            Ring stage;
            unsigned int claim = claim0, ahead = 0;   // the first chunk was claimed before theta arrived
            for (int j = 0;; ++j) {
                const bool have = claim < (unsigned int)n_chunks;
                GlmChunk ch{};
                if (have) ch = chunks[claim];
                if (lane == 0) {
                    ring[j & (kRing - 1)] = have ? make_int4(ch.seg, ch.first_tile * kTileM, ch.n_tiles, 0) : make_int4(-1, 0, 0, 0);
                    mbar_arrive(&bar_ring[j & (kRing - 1)]);
                    if (have) ahead = atomicAdd(work_counter, 1u);   // next claim: the round trip hides behind this chunk
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
                    if (j == 0 && t == preloaded && lane == 0) fed::stamp(comm, 3);
                    const int row0 = (ch.first_tile + t) * kTileM;
                    unsigned char* dst = smem + (size_t)st * L.stage_bytes;
                    if (elect_one()) {
                        mbar_expect_tx(&bar_full[st], L.stage_bytes);
                        for (int pnl = 0; pnl < panels; ++pnl)
                            tma_load_2d(dst + pnl * kPanelBytes, &tmaps[ch.seg], pnl * kPanel, row0, &bar_full[st]);
                    }
                    __syncwarp();
                    stage.advance(S);
                }
                claim = __shfl_sync(0xffffffffu, ahead, 0);
            }
            if (lane == 0) fed::stamp(comm, 4);
        } else if (warp >= 4) {
            // ================= consumer warpgroups ===============================================
            const int c = (warp >> 2) - 1;          // rows 64c .. 64c + 63 of every tile, gradient features c PP/2 ..
            const int w = warp & 3;                 // warp within the group: accumulator rows 16w .. 16w + 15
            const int q = lane & 3;                 // column pair of the accumulator fragment
            const int ew = warp - 4;                // consumer warp ordinal: LL slot row
            const int NB = PP / 128;                // 64-feature gradient blocks per warpgroup (1..3)
            constexpr int NJ = C8 / 8;              // this thread's chains: k = 8 jc + 2 q + e, jc < NJ, e < 2
            // descriptors: constant fields once, the 14-bit (address >> 4) field added per MMA
            const uint64_t desc_k = make_desc(0, 16, 1024, 1);            // X / Theta^T: K-major, 128B swizzle
            const uint64_t desc_xt = make_desc(0, kPanelBytes, 1024, 1);  // X^T: MN-major view of the X panels
            const uint64_t desc_r = make_desc(0, 128, 2048, 0);           // R: K-major (rows contiguous), no swizzle
            const uint32_t theta_b_a = smem_u32(theta_b);
            const uint32_t x_base_a = smem_u32(smem);
            const uint32_t r_a = smem_u32(r_buf);
            float gacc[3][N2 / 2];
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int v = 0; v < N2 / 2; ++v) gacc[i][v] = 0.f;
            Ring stage;
            uint32_t rb = 0;                        // R buffer of the current tile (alternates)
            for (int j = 0;; ++j) {
                const int4 ch = consumer_chunk(j);
                if (ch.x < 0) break;
                const float* __restrict__ seg_y = segs_g[ch.x].y;   // segment table: global, read once per chunk
                const long long seg_rows = segs_g[ch.x].n_rows;
                const int seg_group = segs_g[ch.x].group;
                const int og = segs_g[ch.x].out_group;               // output block of this chunk's segment
                float ll_acc[2 * NJ], gi_acc[2 * NJ];
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) ll_acc[s] = gi_acc[s] = 0.f;
                for (int t = 0; t < ch.z; ++t) {
                    mbar_wait(&bar_full[stage.idx], stage.phase);
                    const uint32_t x_a = x_base_a + (uint32_t)stage.idx * L.stage_bytes;
                    // ---- MMA #1: eta of this group's 64 rows
                    float eacc[N1 / 2];
#pragma unroll
                    for (int v = 0; v < N1 / 2; ++v) eacc[v] = 0.f;
                    wgmma_fence();
                    for (int pnl = 0; pnl < panels; ++pnl) {
#pragma unroll
                        for (int ks = 0; ks < kPanel / 16; ++ks) {
                            const uint64_t adesc = desc_k | (uint64_t)((x_a + pnl * kPanelBytes + c * 64 * 128 + ks * 32) >> 4);
                            const uint64_t bdesc = desc_k | (uint64_t)((theta_b_a + pnl * (N1 * 128) + ks * 32) >> 4);
                            wgmma_bf16<N1, 0, 0>(eacc, adesc, bdesc, (pnl | ks) ? 1u : 0u);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(eacc);
                    // ---- link, likelihood, residual -> (hi, lo) bf16 columns of R (element (row, n) at
                    // (n / 8) * 2048 + (row / 8) * 128 + (n % 8) * 16 + (row % 8) * 2)
                    unsigned char* rbuf = r_buf + rb * L.r_bytes;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = 64 * c + 16 * w + (lane >> 2) + 8 * h;   // row of the tile
                        const long long grow = (long long)ch.y + (long long)t * kTileM + row;
                        const bool valid = grow < seg_rows;
                        const float y = valid ? __ldg(seg_y + grow) : 0.f;
#pragma unroll
                        for (int jc = 0; jc < NJ; ++jc)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int k = 8 * jc + 2 * q + e;
                                const float eta = (eacc[4 * jc + 2 * h + e] + eacc[4 * (NJ + jc) + 2 * h + e]) +
                                                  eacc[4 * (2 * NJ + jc) + 2 * h + e];
                                float ll = 0.f, r = 0.f;
                                if (valid && k < nch) link_loglik(prm.family, y, eta + icpt[k * G + seg_group], ll, r);
                                ll_acc[2 * jc + e] += ll;
                                gi_acc[2 * jc + e] += r;
                                if (k < N2 / 2) {
                                    const __nv_bfloat16 hi = __float2bfloat16_rn(r);
                                    const __nv_bfloat16 lo = __float2bfloat16_rn(r - __bfloat162float(hi));
                                    unsigned char* p0 = rbuf + ((2 * k) / 8) * 2048 + (row / 8) * 128 + (row % 8) * 2;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k) % 8) * 16) = hi;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k + 1) % 8) * 16) = lo;
                                }
                            }
                    }
                    fence_proxy_async();
                    named_sync(1, 32 * kConsumerWarps);   // R of all 128 rows written
                    // ---- MMA #2: G[this group's features] += X^T . R over the 128 rows of the tile
                    wgmma_fence();
#pragma unroll
                    for (int i = 0; i < 3; ++i)
                        if (i < NB) {
                            const uint32_t xa = x_a + (c * NB + i) * kPanelBytes;
#pragma unroll
                            for (int ks = 0; ks < kTileM / 16; ++ks) {
                                const uint64_t adesc = desc_xt | (uint64_t)((xa + ks * 2048) >> 4);
                                const uint64_t bdesc = desc_r | (uint64_t)((r_a + rb * L.r_bytes + ks * 256) >> 4);
                                wgmma_bf16<N2, 1, 0>(gacc[i], adesc, bdesc, (t | ks) ? 1u : 0u);
                            }
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
#pragma unroll
                    for (int i = 0; i < 3; ++i) fence_regs(gacc[i]);
                    mbar_arrive(&bar_empty[stage.idx]);   // this thread is done with the X stage
                    stage.advance(S);
                    rb ^= 1u;
                }
                // ---- end of the chunk: fold its sums into the CTA's running pairs --------------------
                // per-thread fp32 sums over the chunk's tiles -> fixed butterfly over the 8 lanes that share the
                // chains (double) -> lanes 0..3 add the warp's value to its own slot: every step depends on the
                // chunk only.
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) {
                    double lsum = (double)ll_acc[s], gsum = (double)gi_acc[s];
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
                        gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
                    }
                    const int k = 8 * (s >> 1) + 2 * q + (s & 1);
                    if (lane < 4 && k < nch) {
                        double* slot = ll_slots + 2 * ((((size_t)ew * NOUT + og) * KC + k) * NS1);
                        dd_accumulate(slot, lsum);
                        dd_accumulate(slot + 2 * (1 + seg_group), gsum);
                    }
                }
                // gradient: feature f = 64 (c NB + i) + 16 w + lane / 4 + 8 h, chain k = 4 jn + q, (hi, lo) adjacent
#pragma unroll
                for (int i = 0; i < 3; ++i)
                    if (i < NB) {
#pragma unroll
                        for (int jn = 0; jn < N2 / 8; ++jn)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int f = 64 * (c * NB + i) + 16 * w + (lane >> 2) + 8 * h;
                                const int k = 4 * jn + q;
                                if (k < nch && f < P)
                                    dd_accumulate(out + 2 * (((size_t)og * nch + k) * NV1 + 1 + G + f),
                                                  (double)gacc[i][4 * jn + 2 * h] + (double)gacc[i][4 * jn + 2 * h + 1]);
                            }
                    }
            }
        }

        // ---------------- CTA partial: fold the per-warp LL slots and the intercept gradients ----------
        __syncthreads();
        fed::pdl_trigger();   // the next evaluation's CTA may take this SM as soon as we exit
        if (threadIdx.x == 0) fed::stamp(comm, 5);
        // layout per (output block, chain): [LL, gi[G], g[P]] as (hi, lo) pairs; g[] was accumulated in place,
        // LL and gi[] are the per-warp slots summed in warp order
        for (int i = threadIdx.x; i < NOUT * nch * NS1; i += blockDim.x) {
            const int j = i % NS1, k = (i / NS1) % nch, o = i / (NS1 * nch);
            double hi = 0.0, lo = 0.0;
            for (int w = 0; w < kConsumerWarps; ++w) {
                const double* slot = ll_slots + 2 * ((((size_t)w * NOUT + o) * KC + k) * NS1 + j);
                fed::dd_add(hi, lo, slot[0], slot[1]);
            }
            out[2 * (((size_t)o * nch + k) * NV1 + j)] = hi;
            out[2 * (((size_t)o * nch + k) * NV1 + j) + 1] = lo;
        }
        if (threadIdx.x == 0) fed::stamp(comm, 6);
    } else if (warp == 0) {
        // nothing will be computed (stop / idle): the early loads still have to land before the CTA may exit
        for (int t = 0; t < preloaded; ++t) mbar_wait(&bar_full[t], 0u);
    }
    __syncthreads();
    const unsigned long long status = *pipeline_fault() ? B200FED_ERR_PIPELINE : 0ull;
    const bool fin = fed::epilogue_t<true>(comm, pro, status, row_doubles, comm.group_partials);
    if (fin && threadIdx.x == 0) *work_counter = 0u;   // every CTA has stopped claiming: ready for the next launch
}

}  // namespace tc

// ------------------------------------------------------------------ host side
namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
int chains_bucket(int k) { return k <= 1 ? 1 : (k <= 4 ? 4 : (k <= 8 ? 8 : (k <= 16 ? 16 : 0))); }
}  // namespace

// Builds one TMA descriptor per segment ([n_rows, P] bf16, box = 64 features x 128 rows, 128B swizzle) and
// the chunk table.
extern "C" int b200_glm_tc_prepare(const GlmSegment* segs_host, int n_segments, const GlmParams* prm, int sm_count,
                                   void** tmaps_dev, void** chunks_dev, int* n_chunks) {
    if (prm->n_features % 8 != 0 || prm->n_features > 384 || prm->n_features < 8) return -11;   // padded to 128s by TMA
    if (chains_bucket(prm->n_chains) == 0) return -13;
    if ((prm->ld * 2) % 16 != 0) return -14;
    EncodeTiledFn encode = get_encode();
    if (!encode) return -15;
    for (int s = 0; s < n_segments; ++s)
        if (segs_host[s].n_rows + tc::kTileM >= (1ll << 31)) return -18;   // row coordinates are 32-bit
    CUtensorMap* host = new CUtensorMap[n_segments];
    for (int s = 0; s < n_segments; ++s) {
        if (((uintptr_t)segs_host[s].X & 15) != 0) { delete[] host; return -16; }
        cuuint64_t dims[2] = {(cuuint64_t)prm->n_features, (cuuint64_t)segs_host[s].n_rows};
        cuuint64_t strides[1] = {(cuuint64_t)prm->ld * 2};
        cuuint32_t box[2] = {(cuuint32_t)tc::kPanel, (cuuint32_t)tc::kTileM};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&host[s], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(segs_host[s].X), dims, strides,
                            box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { delete[] host; return -17; }
    }
    if (*tmaps_dev) cudaFree(*tmaps_dev);
    cudaError_t e = cudaMalloc(tmaps_dev, sizeof(CUtensorMap) * n_segments);
    if (e == cudaSuccess) e = cudaMemcpy(*tmaps_dev, host, sizeof(CUtensorMap) * n_segments, cudaMemcpyHostToDevice);
    delete[] host;
    if (e != cudaSuccess) return (int)e;
    const std::vector<GlmChunk> chunks = build_chunks(segs_host, n_segments, sm_count > 0 ? sm_count : 132, tc::kTileM, 2,
                                                        tc::kMaxChunk, tc::kMinChunk);
    if (*chunks_dev) cudaFree(*chunks_dev);
    e = cudaMalloc(chunks_dev, sizeof(GlmChunk) * (chunks.size() + 1));
    if (e == cudaSuccess) e = cudaMemcpy(*chunks_dev, chunks.data(), sizeof(GlmChunk) * chunks.size(), cudaMemcpyHostToDevice);
    *n_chunks = (int)chunks.size();
    return e == cudaSuccess ? 0 : (int)e;
}

// The chunk table for given segment sizes (host only; tests/test_chunk_schedule.py).  Writes up to max_chunks
// triples (seg, first_tile, n_tiles) and returns the number of chunks.
extern "C" int b200_glm_tc_chunk_table(const long long* n_rows, int n_segments, int sm_count, int multiple, int max_chunk,
                                       int min_chunk, int* out, int max_chunks) {
    std::vector<GlmSegment> segs(n_segments);
    for (int s = 0; s < n_segments; ++s) segs[s].n_rows = n_rows[s];
    const std::vector<GlmChunk> chunks = build_chunks(segs.data(), n_segments, sm_count, tc::kTileM, multiple, max_chunk, min_chunk);
    for (size_t i = 0; i < chunks.size() && (int)i < max_chunks; ++i) {
        out[3 * i + 0] = chunks[i].seg;
        out[3 * i + 1] = chunks[i].first_tile;
        out[3 * i + 2] = chunks[i].n_tiles;
    }
    return (int)chunks.size();
}

// doubles in the partial array of the tensor-core kernel: one row of (hi, lo) pairs + per-warp LL slots per CTA
extern "C" size_t b200_glm_tc_partial_row_doubles(int n_vals, int n_chains, int n_out, int n_groups) {
    return tc::partial_row_doubles(n_vals, chains_bucket(n_chains), n_out > 0 ? n_out : 1, n_groups);
}

extern "C" int b200_launch_glm_tc(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, const void* tmaps,
                                  const void* chunks_dev, int n_chunks, unsigned int* work_counter, int grid,
                                  cudaStream_t stream) {
    const int kc = chains_bucket(prm->n_chains);
    if (kc == 0) return -1;
    const CUtensorMap* maps = reinterpret_cast<const CUtensorMap*>(tmaps);
#define LAUNCH_TC(KC)                                                                                              \
    do {                                                                                                           \
        const tc::SmemLayout L = tc::smem_layout((prm->n_features + 127) & ~127, tc::Cfg<KC>::N1, tc::Cfg<KC>::N2, comm->n_theta,  \
                                                 prm->n_groups, KC);                                               \
        if (L.stages < 2) return -2;                                                                               \
        cudaFuncSetAttribute(tc::fed_glm_tc_kernel<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total); \
        cudaLaunchConfig_t cfg{};                                                                                  \
        cfg.gridDim = dim3(grid);                                                                                  \
        cfg.blockDim = dim3(tc::kThreads);                                                                         \
        cfg.dynamicSmemBytes = L.total;                                                                            \
        cfg.stream = stream;                                                                                       \
        cudaLaunchAttribute attr[1];                                                                               \
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                           \
        attr[0].val.programmaticStreamSerializationAllowed = 1;                                                    \
        cfg.attrs = attr;                                                                                          \
        cfg.numAttrs = tc::use_pdl() ? 1 : 0;                                                                      \
        cudaLaunchKernelEx(&cfg, tc::fed_glm_tc_kernel<KC>, *comm, segs_dev, *prm, maps,                           \
                           reinterpret_cast<const GlmChunk*>(chunks_dev), n_chunks, work_counter);                 \
    } while (0)
    if (kc == 1) LAUNCH_TC(1);
    else if (kc == 4) LAUNCH_TC(4);
    else if (kc == 8) LAUNCH_TC(8);
    else LAUNCH_TC(16);
#undef LAUNCH_TC
    return (int)cudaGetLastError();
}
