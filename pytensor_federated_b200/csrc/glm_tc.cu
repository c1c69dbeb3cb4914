// Federated GLM log-likelihood + gradient on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Per 128-row tile of the bf16 design matrix X (read from HBM exactly ONCE per evaluation):
//
//   TMA        X[128 x P] -> smem, 128B-swizzled 64-feature panels (cp.async.bulk.tensor), and the tile's
//              128 responses (offsets, weights) -> the stage's row slot, on the same mbarrier
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
// Roles: warp 0 = TMA producer (packed X: warps 1-3 and 12-15 decode); consumer warpgroups 1 and 2 (warps 4-11), which
// setmaxnreg gives 168 registers per thread against 88 for warpgroups 0 and 3, share every tile: warpgroup c
// computes eta / the residuals of rows 64c .. 64c + 63 and the gradient of features c P/2 .. (c + 1) P/2 - 1,
// so every gradient value has one owner thread.  One 256-thread barrier per tile publishes R; the two R
// buffers alternate, so a buffer is rewritten only after both warpgroups have passed the next tile's barrier.
// The federation prologue/epilogue (theta broadcast, NVLink reduce) is fed_comm.cuh.
//
// Workload: BASELINE.json "federated logistic GLM, 10M rows x 256 features per shard, bf16".
#include <cstring>
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
constexpr int kThreads = 512;        // warpgroup 0: TMA producer (warp 0), packed-X decoders (warps 1 to 3);
                                     // warpgroups 1, 2: consumers; warpgroup 3: packed-X decoders
constexpr int kRegs = 65536 / kThreads;   // registers per thread at launch (128), and in the CTA's shared code
constexpr int kConsumerRegs = 168;   // registers per thread of the consumer warpgroups in their role (setmaxnreg) ...
constexpr int kOtherRegs = 88;       // ... and of warpgroups 0 and 3 in theirs: 256 x 168 + 256 x 88 = 65536
static_assert(256 * kConsumerRegs + 256 * kOtherRegs == 65536, "the register split must fill the register file");
constexpr int kConsumerWarps = 8;
constexpr int kMaxChunk = 32;        // tiles per chunk at most (= tiles accumulated in fp32 registers before a flush)
constexpr int kMinChunk = 4;
constexpr int kRing = 16;            // published chunks the consumers may lag behind (needs only ~3)
constexpr int kLLRows = 16;          // per-warp log-likelihood slot rows (>= kConsumerWarps)

// Packed X (GlmParams::packed_x).  A bf16 value is [sign | exponent 8 | mantissa 7]; its high byte (sign and the upper
// 7 exponent bits) takes few values on real data, its low byte is close to random.  Each (128-row tile, 64-feature
// panel) is one kXBlock block: the 8192 low bytes in row-major order, then 8192 4-bit codes (two per byte, the even
// feature in the low nibble), code c < 15 standing for the high byte in entry c of the segment's table (entry 0 is
// 0x00, which padding uses) and 15 for an exception.  A tile's kXFoot-byte footer holds the exception count and up
// to kXMaxExceptions words (position in the tile << 8 | high byte), position = panel * 8192 + row * 64 + feature.
// The producer (warp 0) streams the blocks into a ring of kXSlots slots with cp.async.bulk; warps 1 to 3 and 12 to 15
// decode each panel into the 128B-swizzled image TMA would have written, so the consumers see the same stage bytes.
constexpr int kXBlock = kTileM * kPanel * 3 / 2;   // 12 KB
constexpr int kXFoot = 256;
constexpr int kXMaxExceptions = kXFoot / 4 - 1;
constexpr int kXSlots = 6;                           // compressed panel slots at most
constexpr int kDecThreads = 224;                     // warps 1 to 3 and 12 to 15

// prmt.b32 (byte permute; selector nibble bit 3 replicates the sign of the selected byte)
__host__ __device__ __forceinline__ uint32_t x12_prmt(uint32_t a, uint32_t b, uint32_t s) {
#ifdef __CUDA_ARCH__
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(s));
    return r;
#else
    const uint64_t v = (uint64_t)b << 32 | a;
    uint32_t r = 0;
    for (int k = 0; k < 4; ++k) {
        const uint32_t sel = (s >> (4 * k)) & 0xFu;
        uint32_t byte = (uint32_t)(v >> (8 * (sel & 7u))) & 0xFFu;
        if (sel & 8u) byte = (byte & 0x80u) ? 0xFFu : 0u;
        r |= byte << (8 * k);
    }
    return r;
#endif
}
// Eight consecutive values of a row: low bytes lo (values 0-3 in .x, 4-7 in .y), codes c (nibble k: value k), table t
// (entry 4 q + b in byte b of t[q]) -> the 8 bf16 values as one 16-byte chunk.  Codes index entries 0-7 (t[0], t[1])
// or 8-15 (t[2], t[3]) with their low 3 bits; the per-byte select on bit 3 comes from a sign-replicating prmt of the
// code word's bytes (c << 4 holds bit 3 of the even nibbles in its byte MSBs, c that of the odd ones).
__host__ __device__ __forceinline__ uint4 x12_decode8(uint2 lo, uint32_t c, const uint32_t (&t)[4]) {
    const uint32_t w = c << 4;
    const uint32_t s0 = c & 0x7777u, s1 = (c >> 16) & 0x7777u;
    const uint32_t m0 = x12_prmt(w, c, 0xD9C8u), m1 = x12_prmt(w, c, 0xFBEAu);
    const uint32_t h0 = (x12_prmt(t[0], t[1], s0) & ~m0) | (x12_prmt(t[2], t[3], s0) & m0);
    const uint32_t h1 = (x12_prmt(t[0], t[1], s1) & ~m1) | (x12_prmt(t[2], t[3], s1) & m1);
    uint4 r;
    r.x = x12_prmt(lo.x, h0, 0x5140u);
    r.y = x12_prmt(lo.x, h0, 0x7362u);
    r.z = x12_prmt(lo.y, h1, 0x5140u);
    r.w = x12_prmt(lo.y, h1, 0x7362u);
    return r;
}
// Byte offset in the decoded (128B-swizzled) tile of chunk i = row * 8 + j of a panel
__host__ __device__ __forceinline__ uint32_t x12_chunk_offset(int i) { return (i >> 3) * 128 + (((i & 7) ^ ((i >> 3) & 7)) << 4); }
// Byte offset of the high byte of the value at an exception position (panel * 8192 + row * 64 + feature)
__host__ __device__ __forceinline__ uint32_t x12_high_byte_offset(uint32_t pos) {
    const uint32_t pnl = pos >> 13, row = (pos >> 6) & 127, f = pos & 63;
    return pnl * kPanelBytes + row * 128 + ((((f >> 3) ^ (row & 7)) << 4) | ((f & 7) << 1)) + 1;
}

struct SmemLayout {
    uint32_t stages, stage_bytes, off_theta_b, theta_b_bytes, off_r, r_bytes, off_rows, row_bytes, off_theta_f,
        off_disp, off_ring, off_bars, total, preload, xslots, xslot_bytes, off_x, off_xfoot;
};
// chain_words: per-chain fp32 constants kept in shared memory next to the chunk's intercept column (kDispWords for
// the dispersion families, else 0);
// row_arrays: fp32 per-row arrays a tile carries (y, and the offsets / weights the launch has: 1 to 3)
// packed: X comes packed (kXBlock blocks): two bf16 stages, then as many compressed panel slots as fit (xslots, at most
// kXSlots; fewer than 2 means the shape cannot run packed), each a block plus the footer and row data of its tile.
// theta (fp32) is staged in the two bf16 stages as in the unpacked layout, so a theta larger than both (many groups
// and chains) gets no slots: such a shape reads X itself, with its 3 or 4 stages
__host__ __device__ inline SmemLayout smem_layout(int P, int n1, int n2, int n_theta, int chain_words, int chains,
                                                  int row_arrays, bool packed = false) {
    SmemLayout L;
    const uint32_t panels = P / kPanel;
    L.stage_bytes = panels * kPanelBytes;
    L.theta_b_bytes = panels * n1 * 128;
    L.r_bytes = kTileM * n2 * 2;
    // the row slot of a stage (its tile's y, offset, weight) lies outside the ring, whose last stage the fp32
    // theta staging aliases; it is paid for per stage when the stage count is chosen
    L.row_bytes = (uint32_t)row_arrays * kTileM * 4;
    // theta (fp32) is staged inside the TMA stage ring and is dead once the bf16 B operand and the intercept
    // table are built, so it costs no shared memory of its own.
    const uint32_t bars_bytes = packed ? 256 : 192;
    const uint32_t fixed = L.theta_b_bytes + 2 * L.r_bytes + ((chains * (1 + chain_words) * 4 + 15) & ~15) + kRing * 24 +
                           bars_bytes + (packed ? 2 * kXFoot : 0) + 1024 /*alignment slack*/;
    uint32_t stages = (227u * 1024u - fixed) / (L.stage_bytes + L.row_bytes);
    if (stages > 4) stages = 4;
    L.xslots = 0;
    L.xslot_bytes = kXBlock + kXFoot + L.row_bytes;
    if (packed) {
        const uint32_t two = fixed + 2 * (L.stage_bytes + L.row_bytes);
        stages = 2;
        if (two <= 227u * 1024u && (uint32_t)n_theta * 4u <= 2u * L.stage_bytes) {
            const uint32_t fit = (227u * 1024u - two) / L.xslot_bytes;
            L.xslots = fit < (uint32_t)kXSlots ? fit : (uint32_t)kXSlots;
        }
    }
    L.stages = stages;
    uint32_t o = stages * L.stage_bytes;
    L.off_theta_b = o; o += L.theta_b_bytes;
    L.off_r = o; o += 2 * L.r_bytes;
    L.off_rows = o; o += stages * L.row_bytes;   // 512-byte multiples: 16-byte aligned like every TMA destination
    L.off_x = o; o += L.xslots * L.xslot_bytes;   // 256-byte multiples
    L.off_xfoot = o; o += packed ? 2 * kXFoot : 0;
    // theta (fp32) sits in the LAST stage when it fits into one: the TMA warp fills the first stages - 1 stages
    // with this CTA's first tiles BEFORE theta has arrived (`preload`), the last stage is free once the B
    // operand is built.  (larger theta: stage 0 onwards, needs n_theta * 4 <= stages * stage_bytes, no preload)
    const bool theta_in_last = (uint32_t)n_theta * 4u <= L.stage_bytes && stages >= 2;
    L.off_theta_f = theta_in_last ? (stages - 1) * L.stage_bytes : 0;
    L.preload = theta_in_last ? stages - 1 : 0;
    if (packed) L.preload = L.xslots;   // compressed slots never hold theta: all of them may fill early (panel loads)
    L.off_disp = o; o += (chains * (1 + chain_words) * 4 + 15) & ~15;   // intercept column, then the constants
    L.off_ring = o; o += kRing * 24;   // published chunks + one mbarrier per ring slot
    L.off_bars = o; o += bars_bytes;
    L.total = o + 1024;
    return L;
}

// fp32 arrays in a stage's row slot (host and device agree through this): y, then the offsets and the weights
// when ROWS and some segment of the launch has them (GlmParams::row_data)
__host__ __device__ inline int row_arrays(bool rows, int row_data) {
    return 1 + (rows && (row_data & kGlmRowOffsets) ? 1 : 0) + (rows && (row_data & kGlmRowWeights) ? 1 : 0);
}

// The kernel's template parameters: KC = columns per launch (the K bucket 1, 4, 8 or 16); ROWS = some segment has
// per-row offsets or weights (GlmSegment::offset / weight), so models without them run an instantiation with no trace
// of the extra loads; E = the epilogue, which turns a row's eta into its ll and r (epilogue() maps each family code):
//   Scalar      families 0 to 2 (link_loglik), one column per chain.
//   Softmax     the multinomial family: its C classes ride along N as "virtual chains", column v = k C + c is class c
//               of chain k, and the columns of one row are coupled only through the log-sum-exp of
//               tc::softmax_loglik.  At least two columns, so no KC = 1 instance.
//   Dispersion  a learned dispersion parameter (tc::gaussian_scale_loglik / tc::negbin_loglik): theta rows have stride
//               G + P + 1, the intercept table is followed by kDispWords per-chain constants, the epilogue produces a
//               third per-row value q = dll/dlog_dispersion next to ll and r, and each chain's output block is
//               [LL, gi[G], g[P], dlog_dispersion].
//   Ordinal     the cumulative-logit family: its C - 1 cutpoints ride along N like the multinomial classes, column
//               v = k (C - 1) + j is cutpoint j of chain k, its intercept table row holds intercept - c_j (packed by
//               the host), so MMA #1 gives z_j = eta - c_j, and the columns of one row are coupled only through
//               tc::ordinal_loglik.
//   Survival    the right-censored survival families (tc::weibull_loglik / tc::lognormal_loglik): Dispersion's layout,
//               each row's event taken from the sign of its y (+t event, -t censored; log |y| computed once per row).
//   Hvp         Hessian-vector products of families 0 to 2 (GlmParams::family carries kGlmHvp, masked off for the
//               family branch): pair p runs as column 2p (theta_p, the Scalar epilogue unchanged) and column 2p + 1 (a
//               direction v_p: the host packs theta row 2p + 1 = (v_intercept, v_beta), so the intercept table's odd
//               rows are v_intercept), whose epilogue writes ll = 0 and r = w h(eta_2p) u with u its own eta without
//               the offset; its output block is then [0, (H v)_intercept[G], (H v)_beta[P]].  Both columns of a pair
//               sit in one thread (e = 0 and e = 1).  No KC = 1 instance.
//   ZeroInflated      the zero-inflated Poisson family (tc::zero_inflated_loglik over link_loglik): pair p runs as
//                     column 2p (the count predictor eta: theta row (intercept, beta), the only one that takes the
//                     offset) and column 2p + 1 (the zero logit zeta: theta row (zi_intercept, zi_beta)), in one thread
//                     as in Hvp.  Both predictors are formed before either column's values: column 2p gets the pair's
//                     ll and r = dll/deta, column 2p + 1 ll = 0 and r = dll/dzeta, so the intercept sums, the (hi, lo)
//                     split and MMA #2 give both predictors' gradients.  No KC = 1 instance.
//   ZeroInflatedDisp  the zero-inflated negative binomial: ZeroInflated over negbin_loglik, with Dispersion's theta and
//                     output layout (both theta rows of a pair end in log alpha; the table of column 2p is used, q
//                     comes from column 2p and column 2p + 1 writes q = 0).
//   Positive          the positive-response families with a log link to the mean (tc::gamma_loglik /
//                     tc::inverse_gaussian_loglik): Dispersion's layout with log_dispersion = log shape; log y (and
//                     1 / y) computed once per row and shared by its chains, the family a launch-uniform branch.
//   LocationScale     the Gaussian location-scale family (tc::location_scale_loglik): ZeroInflated's pair plumbing,
//                     with column 2p the mean mu (theta row (intercept, beta), the only one that takes the offset) and
//                     column 2p + 1 s = log sigma (theta row (sigma_intercept, sigma_beta)); column 2p gets ll and
//                     dll/dmu, column 2p + 1 ll = 0 and dll/ds.  No KC = 1 instance.
//   StudentT          the Student-t family (tc::student_t_loglik): LocationScale with ZeroInflatedDisp's theta and
//                     output layout (both theta rows of a pair end in log nu; the table of column 2p is used, q =
//                     dll/dlog_nu comes from column 2p and column 2p + 1 writes q = 0).
//   Beta              beta regression for proportions in (0, 1) (tc::beta_loglik): Dispersion's layout with
//                     log_dispersion = log precision; log y and log(1 - y) computed once per row and shared by its
//                     chains.
// Column layouts follow the wgmma accumulator fragment (thread lane owns columns 8j + 2 (lane % 4) + {0, 1}), so
// that one thread holds every term of the chains it works on.
enum class Epi {
    Scalar, Softmax, Dispersion, Ordinal, Survival, Hvp, ZeroInflated, ZeroInflatedDisp, Positive, LocationScale, StudentT,
    Beta
};

// What the host and the kernel's shared code need to know about an epilogue
struct EpiTraits {
    bool disp;           // theta rows of stride G + P + 1, kDispWords per-chain constants (chain_constants), q
    bool pair;           // chain k is the column pair (2k, 2k + 1), both predictors formed in one thread (not Hvp)
    bool two_columns;    // at least two columns: no KC = 1 instance
    bool group_panels;   // packed X: the decoders' registers allow two panels per load group
};
__host__ __device__ constexpr EpiTraits traits(Epi e) {
    switch (e) {   // {disp, pair, two_columns, group_panels}
        case Epi::Softmax: case Epi::Hvp: return {false, false, true, true};
        case Epi::Dispersion: case Epi::Survival: case Epi::Positive: return {true, false, false, true};
        case Epi::Ordinal: return {false, false, false, false};
        case Epi::ZeroInflated: case Epi::LocationScale: return {false, true, true, true};
        case Epi::ZeroInflatedDisp: case Epi::StudentT: return {true, true, true, true};
        case Epi::Beta: return {true, false, false, false};
        default: return {false, false, false, true};   // Scalar
    }
}

// The per-chain constants of a traits(E).disp epilogue from the chain's log_dispersion ld
template <Epi E>
__device__ __forceinline__ void chain_constants(int family, float ld, float* t) {
    if constexpr (E == Epi::Survival) survival_constants(ld, t);
    else if constexpr (E == Epi::Positive) positive_constants(family, ld, t);
    else if constexpr (E == Epi::StudentT) student_t_constants(ld, t);
    else if constexpr (E == Epi::Beta) beta_constants(ld, t);
    else dispersion_constants(family, ld, t);   // Dispersion; ZeroInflatedDisp: family 10's table is family 5's
}

constexpr Epi epilogue(int family) {
    if (family & kGlmHvp) return Epi::Hvp;
    switch (family) {
        case kGlmMultinomial: return Epi::Softmax;
        case kGlmGaussianScale: case kGlmNegBinomial: return Epi::Dispersion;
        case kGlmOrdinal: return Epi::Ordinal;
        case kGlmWeibull: case kGlmLogNormal: return Epi::Survival;
        case kGlmZeroInflatedPoisson: return Epi::ZeroInflated;
        case kGlmZeroInflatedNegBinomial: return Epi::ZeroInflatedDisp;
        case kGlmGamma: case kGlmInverseGaussian: return Epi::Positive;
        case kGlmGaussianLocationScale: return Epi::LocationScale;
        case kGlmStudentT: return Epi::StudentT;
        case kGlmBeta: return Epi::Beta;
        default: return Epi::Scalar;
    }
}
static_assert([] {
    for (int code = 0; code <= kGlmBeta; ++code)
        if (traits(epilogue(code)).disp != glm_family(code).dispersion) return false;
    return true;
}(), "the epilogue's theta and output layout must match the family's");

// Column layout of the K bucket kc
struct Cfg {
    int C8;   // chain columns per theta term
    int N1;   // eta: term t of chain k in column t * C8 + k
    int N2;   // residual: (hi, lo) of chain k in columns 2k, 2k + 1
};
__host__ __device__ constexpr Cfg cfg(int kc) {
    return {kc <= 8 ? 8 : 16, 3 * (kc <= 8 ? 8 : 16), ((2 * kc + 7) / 8) * 8};
}

// doubles per CTA row of the partial array: (hi, lo) pairs of the n_vals outputs, then the per-warp slots of
// the values that a whole warp contributes to — [kLLRows][n_out][KC][1 + G + disp]: log-likelihood, the G
// intercept gradients and (disp = 1: families with a dispersion parameter) its gradient, of every (output block, chain)
// — the part the launch sums (`partial_sum_doubles`) —, then the CTA's intercept table [KC][G] as floats, padded to
// an even number of doubles so that every row stays 16-byte aligned
__host__ __device__ constexpr size_t partial_sum_doubles(int n_vals, int kc, int n_out, int n_groups, int disp = 0) {
    return 2 * ((size_t)n_vals + (size_t)kLLRows * n_out * kc * (1 + n_groups + disp));
}
__host__ __device__ constexpr size_t partial_row_doubles(int n_vals, int kc, int n_out, int n_groups, int disp = 0) {
    return partial_sum_doubles(n_vals, kc, n_out, n_groups, disp) + ((size_t)kc * n_groups + 3) / 4 * 2;
}

// Work is handed out in CHUNKS of consecutive tiles of one segment (host-built table: 32 tiles while much
// work is left, shrinking to 4 towards the end; always an even number, a segment with an odd tile count
// gets one empty tile).  The TMA warp claims chunks from a global counter and publishes them to the other
// roles through a small shared-memory ring, so CTAs on faster SMs simply take more chunks: no CTA waits on
// a statically assigned straggler.  Everything a chunk contributes (fp32 register accumulation over its tiles,
// per-thread fp32 sums) depends on the chunk alone, and chunk results are combined as double-double pairs
// (fed::dd_add), so the evaluation stays reproducible although the assignment is not.
template <int KC, bool ROWS, Epi E>
__global__ void __launch_bounds__(kThreads, 1)
fed_glm_tc_kernel(FedComm comm, const GlmSegment* __restrict__ segs_g, GlmParams prm, const CUtensorMap* __restrict__ tmaps,
                  const GlmChunk* __restrict__ chunks, int n_chunks, unsigned int* __restrict__ work_counter) {
    constexpr bool SOFTMAX = E == Epi::Softmax, DISP = traits(E).disp, ORD = E == Epi::Ordinal,
                   SURV = E == Epi::Survival, HVP = E == Epi::Hvp, POS = E == Epi::Positive,
                   ZNB = E == Epi::ZeroInflatedDisp, STT = E == Epi::StudentT, BT = E == Epi::Beta;
    constexpr int C8 = cfg(KC).C8;
    constexpr int N1 = cfg(KC).N1;
    constexpr int N2 = cfg(KC).N2;
    extern __shared__ unsigned char smem_dyn[];
    // 1 KB alignment (128B-swizzled TMA tiles) by offsetting INSIDE the shared array: the pointer keeps its
    // shared address space, so the compiler emits LDS / STS instead of generic LD / ST for everything below
    unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);

    const int P = prm.n_features;     // real number of features (theta / result layout)
    const int PP = (P + 127) & ~127;  // features the tile is padded to: TMA zero-fills the columns past P, their
                                      // Theta rows are zero and their gradient rows are never stored
    const int G = prm.n_groups;
    const int panels = PP / kPanel;
    // row slot of a stage: y, then the offsets and the weights when some segment of the launch has them
    const int o_slot = 1, w_slot = ROWS && (prm.row_data & kGlmRowOffsets) ? 2 : 1;
    const bool PK = prm.packed_x != 0;   // X packed: warp 0 loads compressed panels, warps 1 to 3 and 12 to 15 decode them
    const SmemLayout L = smem_layout(PP, N1, N2, comm.n_theta, DISP ? kDispWords : 0, KC, row_arrays(ROWS, prm.row_data), PK);
    const int S = (int)L.stages;
    const int nch = prm.n_chains < KC ? prm.n_chains : KC;  // chains actually present in theta
    const int NV1 = 1 + G + P + DISP; // outputs per chain: [LL, gi[G], g[P]] (DISP: and dlog_dispersion)

    unsigned char* theta_b = smem + L.off_theta_b;
    unsigned char* r_buf = smem + L.off_r;
    float* theta_f = reinterpret_cast<float*>(smem + L.off_theta_f);  // valid until the setup barrier only
    float* icpt = reinterpret_cast<float*>(smem + L.off_disp);        // [KC]: intercepts of the current chunk's group
    float* disp = icpt + KC;                                            // DISP: [KC][kDispWords] per-chain constants
    int4* ring = reinterpret_cast<int4*>(smem + L.off_ring);          // (segment or -1, first row, tiles, group)
    uint64_t* bar_ring = reinterpret_cast<uint64_t*>(smem + L.off_ring + kRing * 16);   // slot j % kRing: chunk j published
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    uint64_t* bar_full = bars;            // [4] X stage landed
    uint64_t* bar_empty = bars + 4;       // [4] X stage consumed by both consumer warpgroups (bars + 128 B: chunk decision)
    uint64_t* bar_xfull = bars + 20;      // PK: [kXSlots] compressed panel landed (bars + 144 B: the decoders' chunk decision)
    uint64_t* bar_xempty = bars + 20 + kXSlots;   // PK: [kXSlots] compressed panel decoded

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---------------- theta-independent setup: runs BEFORE the dependency wait inside fed::prologue, i.e. it
    // overlaps with the tail of the previous evaluation when launched with programmatic stream serialization
    if (threadIdx.x == 0) {
        *pipeline_fault() = 0;
        for (int i = 0; i < kRing; ++i) mbar_init(&bar_ring[i], 1);
        // PK: a stage is full once every decoder thread has arrived (its decoded stores fenced for the async proxy)
        for (int i = 0; i < 4; ++i) { mbar_init(&bar_full[i], PK ? kDecThreads : 1); mbar_init(&bar_empty[i], 32 * kConsumerWarps); }
        if (PK)
            for (int i = 0; i < kXSlots; ++i) { mbar_init(&bar_xfull[i], 1); mbar_init(&bar_xempty[i], kDecThreads); }
        fence_barrier_init();
    }
    // tmaps[4 s + a]: X, y, offset, weight of segment s (the last two only where the segment has them)
    if (warp == 0 && lane == 0)
        for (int i = 0; i < prm.n_segments; ++i) {
            tma_prefetch_desc(&tmaps[4 * i]);
            tma_prefetch_desc(&tmaps[4 * i + 1]);
            if (ROWS && segs_g[i].offset) tma_prefetch_desc(&tmaps[4 * i + 2]);
            if (ROWS && segs_g[i].weight) tma_prefetch_desc(&tmaps[4 * i + 3]);
        }
    // One tile into stage st, issued by one lane: the X panels and the tile's row data (y, then, ROWS, offset and
    // weight where the segment has them: bit 0 / bit 1 of `rows`) into the stage's row slot, all counted on full[st].
    // TMA zero-fills rows past the segment's end.
    auto load_tile = [&](int st, int seg, int row0, int rows) {
        const CUtensorMap* m = tmaps + 4 * seg;
        float* slot = reinterpret_cast<float*>(smem + L.off_rows + (size_t)st * L.row_bytes);
        mbar_expect_tx(&bar_full[st], L.stage_bytes + kTileM * 4 * (1 + (rows & 1) + (rows >> 1)));
        for (int pnl = 0; pnl < panels; ++pnl)
            tma_load_2d(smem + (size_t)st * L.stage_bytes + pnl * kPanelBytes, m, pnl * kPanel, row0, &bar_full[st]);
        tma_load_1d(slot, m + 1, row0, &bar_full[st]);
        if (rows & 1) tma_load_1d(slot + o_slot * kTileM, m + 2, row0, &bar_full[st]);
        if (rows & 2) tma_load_1d(slot + w_slot * kTileM, m + 3, row0, &bar_full[st]);
    };
    // PK: panel pnl of tile `tile` of segment seg into compressed slot xs, issued by one lane; with panel 0 come the
    // tile's exception footer and row data (laid out as in a stage's row slot), all counted on xfull[xs]
    auto load_xpanel = [&](int xs, int seg, int tile, int pnl, int rows) {
        unsigned char* dst = smem + L.off_x + (size_t)xs * L.xslot_bytes;
        const GlmSegment& g = segs_g[seg];
        const uint32_t extra = pnl == 0 ? kXFoot + kTileM * 4 * (1 + (rows & 1) + (rows >> 1)) : 0;
        mbar_expect_tx(&bar_xfull[xs], kXBlock + extra);
        bulk_load(dst, static_cast<const unsigned char*>(g.xpack) + ((size_t)tile * panels + pnl) * kXBlock, kXBlock, &bar_xfull[xs]);
        if (pnl == 0) {
            const CUtensorMap* m = tmaps + 4 * seg;
            float* slot = reinterpret_cast<float*>(dst + kXBlock + kXFoot);
            bulk_load(dst + kXBlock, static_cast<const unsigned char*>(g.xfoot) + (size_t)tile * kXFoot, kXFoot, &bar_xfull[xs]);
            tma_load_1d(slot, m + 1, tile * kTileM, &bar_xfull[xs]);
            if (rows & 1) tma_load_1d(slot + o_slot * kTileM, m + 2, tile * kTileM, &bar_xfull[xs]);
            if (rows & 2) tma_load_1d(slot + w_slot * kTileM, m + 3, tile * kTileM, &bar_xfull[xs]);
        }
    };
    // the row arrays of segment seg that the producer loads (bit 0: offset, bit 1: weight)
    auto seg_row_mask = [&](int seg) -> int {
        if constexpr (!ROWS) return 0;
        return (segs_g[seg].offset ? 1 : 0) | (segs_g[seg].weight ? 2 : 0);
    };
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
            const int units = PK ? ch.n_tiles * panels : ch.n_tiles;   // PK: compressed panels, else tiles
            preloaded = units < (int)L.preload ? units : (int)L.preload;
            if (!prm.early_loads) preloaded = 0;
            const int rows = seg_row_mask(ch.seg);
            if (elect_one())
                for (int t = 0; t < preloaded; ++t) {
                    if (PK) load_xpanel(t, ch.seg, ch.first_tile + t / panels, t % panels, rows);
                    else load_tile(t, ch.seg, (ch.first_tile + t) * kTileM, rows);
                }
            __syncwarp();
        }
    }

    // Nothing that lives from here to the CTA's tail may stay in a register across the role loops below: there it
    // would take one of the consumers' registers in their setmaxnreg region, and at K = 16 it would be spilled.  So
    // the prologue's result waits in shared memory (thread 0 writes it, every thread reads it after the barrier before
    // the tail), and this CTA's row of the partial array is recomputed from the launch parameters and the block index
    // where it is used (opaque() keeps the compiler from merging the copies into one long-lived value).
    __shared__ fed::Prologue s_pro;
    bool active;
    {
        const fed::Prologue pro = fed::prologue(comm, theta_f);   // contains __syncthreads()
        if (threadIdx.x == 0) s_pro = pro;
        active = !pro.stop && !pro.timed_out;
    }
    const int NOUT = prm.n_out;       // output blocks (1 = everything summed; else one per node)
    const int NS1 = 1 + G + DISP;     // warp-level values per (block, chain): LL, the G intercept gradients (and q)
    auto row_doubles = [&] { return partial_row_doubles(opaque(comm.n_vals), KC, NOUT, G, DISP); };
    // this CTA's running sums, (hi, lo) pairs
    auto cta_row = [&]() -> double* { return comm.cta_partials + (size_t)blockIdx.x * row_doubles(); };
    // [KC][G] intercepts, in global memory so that the shared memory budget does not grow with G: written in the
    // setup below, read by this CTA only (after __syncthreads), one column into `icpt` per chunk
    auto icpt_table = [&]() -> float* {
        return reinterpret_cast<float*>(cta_row() + partial_sum_doubles(opaque(comm.n_vals), KC, NOUT, G, DISP));
    };
    // [kLLRows][NOUT][KC][NS1] pairs
    auto ll_slots = [&]() -> double* { return cta_row() + 2 * (size_t)opaque(comm.n_vals); };

    if (active) {
        // ---------------- theta-dependent setup --------------------------------------------------
        {
            double* out = cta_row();
            const size_t sum_doubles = partial_sum_doubles(comm.n_vals, KC, NOUT, G, DISP);
            for (size_t i = threadIdx.x; i < sum_doubles / 2; i += blockDim.x) reinterpret_cast<double2*>(out)[i] = make_double2(0.0, 0.0);
        }
        float* const itab = icpt_table();
        for (int i = threadIdx.x; i < KC * G; i += blockDim.x)
            itab[i] = (i / G) < nch ? theta_f[(i / G) * (G + P + DISP) + (i % G)] : 0.f;   // theta row stride G + P (+ 1)
        if constexpr (DISP)
            for (int k = threadIdx.x; k < KC; k += blockDim.x)
                chain_constants<E>(prm.family, k < nch ? theta_f[k * (G + P + 1) + G + P] : 0.f, disp + k * kDispWords);
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
                    const float v = f < P ? theta_f[chain * (G + P + DISP) + G + f] : 0.f;
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
            // the intercepts of the chunk's group (ring entry .w); every reader of the previous column has passed the
            // barrier above
            if (threadIdx.x >= 128 && threadIdx.x < 128 + KC && !*pipeline_fault() && ring[slot].x >= 0)
                icpt[threadIdx.x - 128] = __ldcg(icpt_table() + (threadIdx.x - 128) * G + ring[slot].w);
            named_sync(1, 256);
            return *chunk_decided;
        };

        // Registers go where the work needs them: the consumer warpgroups' epilogues get kConsumerRegs per thread, the
        // producer and the decoders (warpgroups 0 and 3) kOtherRegs.  setmaxnreg is per warpgroup, so each side
        // changes its count at the top of its branch (warp 0 together with warps 1 to 3) and returns to kRegs at its
        // end, before the CTA's shared tail below, on every path (packed or not, and after a stalled pipeline).
        // Warpgroups 0 and 3 take their registers back only after barrier 3, which the consumers reach once they have
        // returned theirs: an idle warpgroup (bf16 X, or a CTA without work) that took them back at once could leave
        // a consumer warpgroup waiting for registers forever, and the other one with it at their named barrier.
        if (warp < 4 || warp >= 12) {
            setmaxnreg<kRegs, kOtherRegs>();
            if (warp == 0) {
                // ================= TMA producer + chunk scheduler ==================================
                // The role loops are warp-uniform (all 32 lanes wait and count); only the issue is predicated on
                // elect.sync, so the compiler keeps addresses / descriptors in uniform registers.
                Ring stage, xs;
                unsigned int claim = claim0, ahead = 0;   // the first chunk was claimed before theta arrived
                for (int j = 0;; ++j) {
                    const bool have = claim < (unsigned int)n_chunks;
                    GlmChunk ch{};
                    if (have) ch = chunks[claim];
                    if (lane == 0) {
                        ring[j & (kRing - 1)] = have ? make_int4(ch.seg, ch.first_tile * kTileM, ch.n_tiles, segs_g[ch.seg].group)
                                                     : make_int4(-1, 0, 0, 0);
                        mbar_arrive(&bar_ring[j & (kRing - 1)]);
                        if (have) ahead = atomicAdd(work_counter, 1u);   // next claim: the round trip hides behind this chunk
                    }
                    __syncwarp();
                    if (!have) break;
                    const int rows = seg_row_mask(ch.seg);
                    for (int t = 0; t < ch.n_tiles && PK; ++t)
                        for (int pnl = 0; pnl < panels; ++pnl) {
                            const int k = t * panels + pnl;
                            if (!(j == 0 && k < preloaded)) {   // else already in flight (early loads)
                                mbar_wait(&bar_xempty[xs.idx], xs.phase ^ 1);
                                if (j == 0 && k == preloaded && lane == 0) fed::stamp(comm, 3);
                                if (elect_one()) load_xpanel(xs.idx, ch.seg, ch.first_tile + t, pnl, rows);
                                __syncwarp();
                            }
                            xs.advance((int)L.xslots);
                        }
                    for (int t = 0; t < ch.n_tiles && !PK; ++t) {
                        const int st = stage.idx;
                        if (j == 0 && t < preloaded) {   // already in flight (early loads)
                            stage.advance(S);
                            continue;
                        }
                        mbar_wait(&bar_empty[st], stage.phase ^ 1);
                        if (j == 0 && t == preloaded && lane == 0) fed::stamp(comm, 3);
                        if (elect_one()) load_tile(st, ch.seg, (ch.first_tile + t) * kTileM, rows);
                        __syncwarp();
                        stage.advance(S);
                    }
                    claim = __shfl_sync(0xffffffffu, ahead, 0);
                }
                if (lane == 0) fed::stamp(comm, 4);
            } else {
                // ================= PK: decoders (warps 1 to 3 and 12 to 15) =============================
                // Per tile: wait for a free stage, decode its panels in order as their compressed slots land (the slot is
                // released right after), copy the footer (double-buffered by tile parity: the barrier below orders every
                // read of buffer b before its next write, two tiles later) and the row data, then patch the exceptions
                // once all 224 threads' stores are in, and arrive on full[stage] after a proxy fence.  Every decoder thread
                // reads every slot (the chunks of a panel are strided over all 224), so every one of them releases it.
                if (PK) {
                    const int td = warp < 4 ? threadIdx.x - 32 : threadIdx.x - (12 * 32 - 96);   // 0 to 95, 96 to 223
                    // panels per load group: 2 where the registers it needs did not push the instantiation into
                    // spills when the whole kernel had one register count (ptxas -v), else 1.  With seven decoder warps
                    // and kOtherRegs of their own, groups of 1 measured slower at K = 1 (docs/KERNELS.md)
                    constexpr int kDecGroup = KC <= 4 && traits(E).group_panels ? 2 : 1;
                    static_assert(kDecGroup <= 2, "a packed launch may have only 2 compressed slots");
                    int4* decided = reinterpret_cast<int4*>(smem + L.off_bars + 144);
                    Ring stage, xs;
                    uint32_t fb = 0;
                    for (int j = 0;; ++j) {
                        // decide each chunk together, as the consumers do: a decoder warp leaving on a stalled pipeline
                        // while the others wait at the barrier below would hang
                        mbar_wait(&bar_ring[j & (kRing - 1)], (uint32_t)((j / kRing) & 1));
                        named_sync(2, kDecThreads);
                        if (td == 0) *decided = *pipeline_fault() ? make_int4(-1, 0, 0, 0) : ring[j & (kRing - 1)];
                        named_sync(2, kDecThreads);
                        const int4 ch = *decided;
                        if (ch.x < 0) break;
                        const uint32_t tab[4] = {segs_g[ch.x].xtab[0], segs_g[ch.x].xtab[1], segs_g[ch.x].xtab[2],
                                                 segs_g[ch.x].xtab[3]};
                        for (int t = 0; t < ch.z; ++t) {
                            mbar_wait(&bar_empty[stage.idx], stage.phase ^ 1);
                            unsigned char* dst = smem + (size_t)stage.idx * L.stage_bytes;
                            int* foot = reinterpret_cast<int*>(smem + L.off_xfoot + fb * kXFoot);
                            // panels in groups of kDecGroup: all of this thread's loads of a group's panels first,
                            // then their decodes and stores.  Two decoder warps share each scheduler but warp 0's (one),
                            // so the shared-memory latency is hidden by those warps and by ILP: a group keeps kDecGroup
                            // panels of loads in flight.  A group holds kDecGroup slots at once: a packed launch has at
                            // least 2 slots (launch() refuses fewer) and 2 or 4 panels, so a group of 2 always fits and
                            // divides the tile.
                            for (int pnl = 0; pnl < panels; pnl += kDecGroup) {
                                constexpr int kPer = (kTileM * 8 + kDecThreads - 1) / kDecThreads;
                                uint2 lo[kDecGroup][kPer];
                                uint32_t cw[kDecGroup][kPer];
                                int xi[kDecGroup];
#pragma unroll
                                for (int h = 0; h < kDecGroup; ++h) {
                                    mbar_wait(&bar_xfull[xs.idx], xs.phase);
                                    const unsigned char* src = smem + L.off_x + (size_t)xs.idx * L.xslot_bytes;
                                    if (pnl + h == 0) {
                                        if (td < kXFoot / 4) foot[td] = reinterpret_cast<const int*>(src + kXBlock)[td];
                                        const float* rsrc = reinterpret_cast<const float*>(src + kXBlock + kXFoot);
                                        float* rdst = reinterpret_cast<float*>(smem + L.off_rows + (size_t)stage.idx * L.row_bytes);
                                        for (int i = td; i < (int)L.row_bytes / 4; i += kDecThreads) rdst[i] = rsrc[i];
                                    }
#pragma unroll
                                    for (int k = 0; k < kPer; ++k) {
                                        const int i = td + k * kDecThreads;
                                        if (k < kPer - 1 || i < kTileM * 8) {
                                            lo[h][k] = reinterpret_cast<const uint2*>(src)[i];
                                            cw[h][k] = reinterpret_cast<const uint32_t*>(src + kTileM * kPanel)[i];
                                        }
                                    }
                                    xi[h] = xs.idx;
                                    xs.advance((int)L.xslots);
                                }
#pragma unroll
                                for (int h = 0; h < kDecGroup; ++h) {
                                    unsigned char* pd = dst + (pnl + h) * kPanelBytes;
#pragma unroll
                                    for (int k = 0; k < kPer; ++k) {
                                        const int i = td + k * kDecThreads;
                                        if (k < kPer - 1 || i < kTileM * 8)
                                            *reinterpret_cast<uint4*>(pd + x12_chunk_offset(i)) = x12_decode8(lo[h][k], cw[h][k], tab);
                                    }
                                    mbar_arrive(&bar_xempty[xi[h]]);
                                }
                            }
                            named_sync(2, kDecThreads);   // the tile's decoded chunks and its footer are in
                            const int n_ex = min(foot[0], kXMaxExceptions);
                            for (int e = td; e < n_ex; e += kDecThreads) {
                                const uint32_t v = (uint32_t)foot[1 + e];
                                if ((v >> 8) < (uint32_t)panels * kTileM * kPanel) dst[x12_high_byte_offset(v >> 8)] = (unsigned char)(v & 0xFFu);
                            }
                            fence_proxy_async();
                            mbar_arrive(&bar_full[stage.idx]);
                            stage.advance(S);
                            fb ^= 1u;
                        }
                    }
                }
            }
            named_sync(3, kThreads);   // every consumer has returned its registers
            setmaxnreg<kOtherRegs, kRegs>();
        } else {
            // ================= consumer warpgroups (warps 4 to 11) ===============================
            setmaxnreg<kRegs, kConsumerRegs>();
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
            // SOFTMAX: chain and class of this thread's columns v = 8 jc + 2 q + e (chain -1: past K C)
            int sm_chain[2 * NJ];
            float sm_cls[2 * NJ];
            int sm_chains = 0;
            if constexpr (SOFTMAX) {
                const int NC = prm.n_classes;
                sm_chains = nch / NC;
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) {
                    const int v = 8 * (s >> 1) + 2 * q + (s & 1);
                    sm_chain[s] = v < nch ? v / NC : -1;
                    sm_cls[s] = (float)(v % NC);
                }
            }
            // ORD: chain and cutpoint of this thread's columns (chain -1: past K (C - 1))
            int od_chain[2 * NJ], od_cut[2 * NJ];
            int od_chains = 0, od_ncut = 1;
            if constexpr (ORD) {
                od_ncut = prm.n_classes - 1;
                od_chains = nch / od_ncut;
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) {
                    const int v = 8 * (s >> 1) + 2 * q + (s & 1);
                    od_chain[s] = v < nch ? v / od_ncut : -1;
                    od_cut[s] = v % od_ncut;
                }
            }
            Ring stage;
            uint32_t rb = 0;                        // R buffer of the current tile (alternates)
            for (int j = 0;; ++j) {
                const int4 ch = consumer_chunk(j);
                if (ch.x < 0) break;
                // segment table: global, read once per chunk; an absent offset / weight reads as 0 / 1 (chunk-uniform)
                const bool has_o = ROWS && segs_g[ch.x].offset != nullptr;
                const bool has_w = ROWS && segs_g[ch.x].weight != nullptr;
                const long long seg_rows = segs_g[ch.x].n_rows;
                const int seg_group = segs_g[ch.x].group;
                const int og = segs_g[ch.x].out_group;               // output block of this chunk's segment
                float ll_acc[2 * NJ], gi_acc[2 * NJ], ds_acc[2 * NJ];   // ds: DISP only (dll/dlog_dispersion)
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) ll_acc[s] = gi_acc[s] = ds_acc[s] = 0.f;
                for (int t = 0; t < ch.z; ++t) {
                    mbar_wait(&bar_full[stage.idx], stage.phase);
                    const uint32_t x_a = x_base_a + (uint32_t)stage.idx * L.stage_bytes;
                    // y, offset, weight of the tile's rows: landed with X (the TMA producer loads them into the stage's slot)
                    const float* row_slot = reinterpret_cast<const float*>(smem + L.off_rows + (size_t)stage.idx * L.row_bytes);
                    // ---- MMA #1: eta of this group's 64 rows
                    float eacc[N1 / 2];
#pragma unroll
                    for (int v = 0; v < N1 / 2; ++v) eacc[v] = 0.f;
                    wgmma_fence();
                    // not unrolled: nvcc's unrolled copies of this runtime-bound loop move accumulator registers
                    // between the wgmmas, and ptxas then waits for each wgmma before issuing the next (C7515)
#pragma unroll 1
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
                    // BT: eta of the thread's columns (the sum of the three bf16 terms), formed once so that the
                    // accumulator fragment is dead during the long per-column evaluations below
                    float bt_eta[2 * 2 * NJ];
                    if constexpr (BT) {
#pragma unroll
                        for (int i = 0; i < 4 * NJ; ++i) {
                            const int h = i / (2 * NJ), jc = (i % (2 * NJ)) >> 1, e = i & 1;
                            bt_eta[i] = (eacc[4 * jc + 2 * h + e] + eacc[4 * (NJ + jc) + 2 * h + e]) +
                                        eacc[4 * (2 * NJ + jc) + 2 * h + e];
                        }
                    }
                    // ---- link, likelihood, residual -> (hi, lo) bf16 columns of R (element (row, n) at
                    // (n / 8) * 2048 + (row / 8) * 128 + (n % 8) * 16 + (row % 8) * 2)
                    unsigned char* rbuf = r_buf + rb * L.r_bytes;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = 64 * c + 16 * w + (lane >> 2) + 8 * h;   // row of the tile
                        const long long grow = (long long)ch.y + (long long)t * kTileM + row;
                        const bool valid = grow < seg_rows;
                        // response, offset and weight of the row
                        const float y = valid ? row_slot[row] : 0.f;
                        float o = 0.f, wt = 1.f;
                        if constexpr (ROWS) {
                            o = valid && has_o ? row_slot[o_slot * kTileM + row] : 0.f;
                            wt = valid && has_w ? row_slot[w_slot * kTileM + row] : 1.f;
                        }
                        // SURV: the row's event and log time, shared by its chains (a row past the segment reads y = 0,
                        // -inf here, and is dropped below; a masked row's NaN is removed by the weight's select)
                        bool sv_event = true;
                        float sv_lt = 0.f;
                        if constexpr (SURV) {
                            sv_event = !signbit(y);
                            sv_lt = logf(fabsf(y));
                        }
                        // POS: log y and 1 / y of the row, shared by its chains (as in SURV, a row past the segment
                        // reads y = 0 and is dropped below, a masked row's NaN or negative y is removed by the weight's
                        // select); 1 / y only for the inverse Gaussian family (launch-uniform)
                        float pv_lt = 0.f, pv_iy = 0.f;
                        if constexpr (POS) {
                            pv_lt = logf(y);
                            if (prm.family == kGlmInverseGaussian) pv_iy = __frcp_rn(y);
                        }
                        // BT: log y and log(1 - y) of the row, shared by its chains (a row past the segment and a masked
                        // row's y outside (0, 1) are dropped below, as in POS)
                        float bt_ly = 0.f, bt_l1y = 0.f;
                        if constexpr (BT) {
                            bt_ly = logf(y);
                            bt_l1y = log1pf(-y);
                        }
                        // SOFTMAX: the row's log-sum-exp per chain over the quad; every lane takes part, whether its
                        // row is valid or not (a row past the segment is dropped below, as in the other families)
                        float sm_ll[2 * NJ], sm_r[2 * NJ];
                        if constexpr (SOFTMAX) {
                            float sm_eta[2 * NJ];
#pragma unroll
                            for (int s = 0; s < 2 * NJ; ++s) {
                                const int jc = s >> 1, e = s & 1;
                                // the intercept table has KC rows but a lane's columns reach 8 NJ - 1 (7 in the
                                // KC = 4 bucket): a column past K C (chain -1, never used) reads row 0, so the
                                // index stays inside the table whatever G is
                                const int k = sm_chain[s] >= 0 ? 8 * jc + 2 * q + e : 0;
                                sm_eta[s] = ((eacc[4 * jc + 2 * h + e] + eacc[4 * (NJ + jc) + 2 * h + e]) +
                                             eacc[4 * (2 * NJ + jc) + 2 * h + e]) + icpt[k];
                                sm_ll[s] = sm_r[s] = 0.f;
                            }
                            softmax_loglik<2 * NJ, KC / 2>(sm_eta, sm_chain, sm_cls, sm_chains, y, sm_ll, sm_r);
                        }
                        // ORD: z = eta - c_j (+ offset, as in ROWS) of every column, coupled per chain over the quad;
                        // every lane takes part, valid row or not.  The label is clamped into [0, C - 1], so a masked
                        // row's NaN or out-of-range y (dropped below) still indexes inside the intercept table.
                        float od_ll[2 * NJ], od_r[2 * NJ];
                        if constexpr (ORD) {
                            float z[2 * NJ];
#pragma unroll
                            for (int s = 0; s < 2 * NJ; ++s) {
                                const int jc = s >> 1, e = s & 1;
                                const int k = od_chain[s] >= 0 ? 8 * jc + 2 * q + e : 0;   // as in SOFTMAX
                                z[s] = ((eacc[4 * jc + 2 * h + e] + eacc[4 * (NJ + jc) + 2 * h + e]) +
                                        eacc[4 * (2 * NJ + jc) + 2 * h + e]) + icpt[k];
                                if constexpr (ROWS) z[s] = __fadd_rn(z[s], o);
                            }
                            const int yi = min(max(__float2int_rz(y), 0), od_ncut);   // NaN -> 0
                            ordinal_loglik<2 * NJ, KC>(z, od_chain, od_cut, od_chains, od_ncut, yi, icpt, 1,
                                                       od_ll, od_r);
                        }
                        if constexpr (BT) {
                            // one column at a time (a rolled loop; its eta and accumulators are picked by selects, so
                            // they stay in registers): beta_loglik is long, and K = 16 has no registers for two of
                            // them in flight.  Each column gets the values and additions of the unrolled loop below.
#pragma unroll 1
                            for (int s = 0; s < 2 * NJ; ++s) {
                                const int k = 8 * (s >> 1) + 2 * q + (s & 1);
                                float eta = 0.f;
#pragma unroll
                                for (int i = 0; i < 2 * NJ; ++i) eta = i == s ? bt_eta[2 * NJ * h + i] : eta;
                                float ll = 0.f, r = 0.f, dq = 0.f;
                                if (valid && k < nch) {
                                    // offset and weight as in ROWS, the weight applied to all three values
                                    float et = eta + icpt[k];
                                    if constexpr (ROWS) et = __fadd_rn(et, o);
                                    beta_loglik(y, bt_ly, bt_l1y, et, disp + k * kDispWords, ll, r, dq);
                                    if constexpr (ROWS) {
                                        apply_weight(wt, ll);
                                        apply_weight(wt, r);
                                        apply_weight(wt, dq);
                                    }
                                }
#pragma unroll
                                for (int i = 0; i < 2 * NJ; ++i) {
                                    ll_acc[i] += i == s ? ll : 0.f;
                                    gi_acc[i] += i == s ? r : 0.f;
                                    ds_acc[i] += i == s ? dq : 0.f;
                                }
                                if (k < N2 / 2) {
                                    const __nv_bfloat16 hi = __float2bfloat16_rn(r);
                                    const __nv_bfloat16 lo = __float2bfloat16_rn(r - __bfloat162float(hi));
                                    unsigned char* p0 = rbuf + ((2 * k) / 8) * 2048 + (row / 8) * 128 + (row % 8) * 2;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k) % 8) * 16) = hi;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k + 1) % 8) * 16) = lo;
                                }
                            }
                        } else {
#pragma unroll
                        for (int jc = 0; jc < NJ; ++jc) {
                            float hv_h = 0.f;   // HVP: h = d2ll / deta2 of the pair's theta column (e = 0), for e = 1
                            // traits(E).pair: the pair's values (columns k0 = 8 jc + 2 q and k0 + 1), from both predictors,
                            // before the column loop; offset and weight as in ROWS (the offset to the first predictor only).
                            // n_chains is even, so k0 < nch covers both columns.
                            float pr_ll = 0.f, pr_r0 = 0.f, pr_r1 = 0.f, pr_q = 0.f;
                            if constexpr (traits(E).pair) {
                                const int k0 = 8 * jc + 2 * q;
                                if (valid && k0 < nch) {
                                    float et = ((eacc[4 * jc + 2 * h] + eacc[4 * (NJ + jc) + 2 * h]) +
                                                eacc[4 * (2 * NJ + jc) + 2 * h]) + icpt[k0];
                                    if constexpr (ROWS) et = __fadd_rn(et, o);
                                    const float zt = ((eacc[4 * jc + 2 * h + 1] + eacc[4 * (NJ + jc) + 2 * h + 1]) +
                                                      eacc[4 * (2 * NJ + jc) + 2 * h + 1]) + icpt[k0 + 1];
                                    if constexpr (E == Epi::LocationScale)
                                        location_scale_loglik(y, et, zt, pr_ll, pr_r0, pr_r1);
                                    else if constexpr (STT)
                                        student_t_loglik(y, et, zt, disp + k0 * kDispWords, pr_ll, pr_r0, pr_r1, pr_q);
                                    else
                                        zero_inflated_loglik<ZNB>(y, et, zt, disp + k0 * kDispWords, pr_ll, pr_r0, pr_r1, pr_q);
                                    if constexpr (ROWS) {
                                        apply_weight(wt, pr_ll);
                                        apply_weight(wt, pr_r0);
                                        apply_weight(wt, pr_r1);
                                        apply_weight(wt, pr_q);
                                    }
                                }
                            }
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int k = 8 * jc + 2 * q + e;
                                const float eta = (eacc[4 * jc + 2 * h + e] + eacc[4 * (NJ + jc) + 2 * h + e]) +
                                                  eacc[4 * (2 * NJ + jc) + 2 * h + e];
                                float ll = 0.f, r = 0.f, dq = 0.f;
                                if (valid && k < nch) {
                                    if constexpr (traits(E).pair) {
                                        // column 2p: the pair's ll, the first predictor's r (and dll/dlog_dispersion);
                                        // 2p + 1: the second predictor's r
                                        ll = e == 0 ? pr_ll : 0.f;
                                        r = e == 0 ? pr_r0 : pr_r1;
                                        dq = e == 0 ? pr_q : 0.f;
                                    } else if constexpr (DISP) {
                                        // offset and weight as in ROWS, the weight applied to all three values
                                        float et = eta + icpt[k];
                                        if constexpr (ROWS) et = __fadd_rn(et, o);
                                        const float* dt = disp + k * kDispWords;   // k < nch <= KC: inside the table
                                        if constexpr (SURV) {
                                            if (prm.family == kGlmWeibull) weibull_loglik(sv_event, sv_lt, et, dt, ll, r, dq);
                                            else lognormal_loglik(sv_event, sv_lt, et, dt, ll, r, dq);
                                        } else if constexpr (POS) {
                                            if (prm.family == kGlmGamma) gamma_loglik(pv_lt, et, dt, ll, r, dq);
                                            else inverse_gaussian_loglik(y, pv_lt, pv_iy, et, dt, ll, r, dq);
                                        } else {
                                            if (prm.family == kGlmGaussianScale) gaussian_scale_loglik(y, et, dt, ll, r, dq);
                                            else negbin_loglik(y, et, dt, ll, r, dq);
                                        }
                                        if constexpr (ROWS) {
                                            apply_weight(wt, ll);
                                            apply_weight(wt, r);
                                            apply_weight(wt, dq);
                                        }
                                    } else if constexpr (ORD) {
                                        // offset already in z; weight as in ROWS
                                        ll = od_ll[2 * jc + e];
                                        r = od_r[2 * jc + e];
                                        if constexpr (ROWS) {
                                            apply_weight(wt, ll);
                                            apply_weight(wt, r);
                                        }
                                    } else if constexpr (SOFTMAX) {
                                        // weight as in ROWS (offsets are rejected for this family)
                                        ll = sm_ll[2 * jc + e];
                                        r = sm_r[2 * jc + e];
                                        if constexpr (ROWS) {
                                            apply_weight(wt, ll);
                                            apply_weight(wt, r);
                                        }
                                    } else if constexpr (HVP) {
                                        // column 2p (e = 0): theta_p, exactly as the scalar families below, plus h at
                                        // its eta; column 2p + 1 (e = 1): the direction v_p, u = x'v_beta + v_intercept
                                        // (no offset: u is linear in v), ll = 0 and r = s = w h u, so that MMA #2 and
                                        // the intercept sums give (H v)_beta and (H v)_intercept
                                        const int fam = prm.family & ~kGlmHvp;
                                        if (e == 0) {
                                            float et = eta + icpt[k];
                                            if constexpr (ROWS) et = __fadd_rn(et, o);
                                            link_loglik(fam, y, et, ll, r);
                                            hv_h = link_curvature(fam, et);
                                            if constexpr (ROWS) {
                                                apply_weight(wt, ll);
                                                apply_weight(wt, r);
                                            }
                                        } else {
                                            r = __fmul_rn(hv_h, eta + icpt[k]);
                                            if constexpr (ROWS) apply_weight(wt, r);
                                        }
                                    } else if constexpr (ROWS) {
                                        // offset after the intercept, weight after the likelihood, both rounded on their
                                        // own (no FMA contraction): w = 1, o = 0 gives the bits of the plain model; a
                                        // zero weight selects 0, so a masked row's non-finite y or o never reaches a sum
                                        link_loglik(prm.family, y, __fadd_rn(eta + icpt[k], o), ll, r);
                                        apply_weight(wt, ll);
                                        apply_weight(wt, r);
                                    } else {
                                        link_loglik(prm.family, y, eta + icpt[k], ll, r);
                                    }
                                }
                                ll_acc[2 * jc + e] += ll;
                                gi_acc[2 * jc + e] += r;
                                if constexpr (DISP) ds_acc[2 * jc + e] += dq;
                                if (k < N2 / 2) {
                                    const __nv_bfloat16 hi = __float2bfloat16_rn(r);
                                    const __nv_bfloat16 lo = __float2bfloat16_rn(r - __bfloat162float(hi));
                                    unsigned char* p0 = rbuf + ((2 * k) / 8) * 2048 + (row / 8) * 128 + (row % 8) * 2;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k) % 8) * 16) = hi;
                                    *reinterpret_cast<__nv_bfloat16*>(p0 + ((2 * k + 1) % 8) * 16) = lo;
                                }
                            }
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
                double* const out = cta_row();
                double* const slots = out + 2 * (size_t)comm.n_vals;
#pragma unroll
                for (int s = 0; s < 2 * NJ; ++s) {
                    double lsum = (double)ll_acc[s], gsum = (double)gi_acc[s], dsum = (double)ds_acc[s];
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
                        gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
                        if constexpr (DISP) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
                    }
                    const int k = 8 * (s >> 1) + 2 * q + (s & 1);
                    if (lane < 4 && k < nch) {
                        double* slot = slots + 2 * ((((size_t)ew * NOUT + og) * KC + k) * NS1);
                        dd_accumulate(slot, lsum);
                        dd_accumulate(slot + 2 * (1 + seg_group), gsum);
                        if constexpr (DISP) dd_accumulate(slot + 2 * (1 + G), dsum);
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
            setmaxnreg<kConsumerRegs, kRegs>();
            named_sync(3, kThreads);
        }

        // ---------------- CTA partial: fold the per-warp LL slots and the intercept gradients ----------
        __syncthreads();
        fed::pdl_trigger();   // the next evaluation's CTA may take this SM as soon as we exit
        if (threadIdx.x == 0) fed::stamp(comm, 5);
        // layout per (output block, chain): [LL, gi[G], g[P]] as (hi, lo) pairs (DISP: then dlog_dispersion);
        // g[] was accumulated in place, LL, gi[] (and dlog_dispersion) are the per-warp slots summed in warp order
        double* const out = cta_row();
        const double* const slots = ll_slots();
        for (int i = threadIdx.x; i < NOUT * nch * NS1; i += blockDim.x) {
            const int j = i % NS1, k = (i / NS1) % nch, o = i / (NS1 * nch);
            double hi = 0.0, lo = 0.0;
            for (int w = 0; w < kConsumerWarps; ++w) {
                const double* slot = slots + 2 * ((((size_t)w * NOUT + o) * KC + k) * NS1 + j);
                fed::dd_add(hi, lo, slot[0], slot[1]);
            }
            const int jo = (DISP && j == 1 + G) ? 1 + G + P : j;   // slot 1 + G: the last value of the block
            out[2 * (((size_t)o * nch + k) * NV1 + jo)] = hi;
            out[2 * (((size_t)o * nch + k) * NV1 + jo) + 1] = lo;
        }
        if (threadIdx.x == 0) fed::stamp(comm, 6);
    } else if (warp == 0) {
        // nothing will be computed (stop / idle): the early loads still have to land before the CTA may exit
        for (int t = 0; t < preloaded; ++t) mbar_wait(PK ? &bar_xfull[t] : &bar_full[t], 0u);
    }
    __syncthreads();
    const unsigned long long status = *pipeline_fault() ? B200FED_ERR_PIPELINE : 0ull;
    const fed::Prologue pro = s_pro;
    // 12 (hi, lo) pairs of loads in flight in the final sums: 16 would not fit the 128 registers of the tail
    const bool fin = fed::epilogue_t<true, 12>(comm, pro, status, row_doubles(), comm.group_partials);
    if (fin && threadIdx.x == 0) *work_counter = 0u;   // every CTA has stopped claiming: ready for the next launch
}

}  // namespace tc

// ------------------------------------------------------------------ host side
namespace {
int chains_bucket(int k) { return k <= 1 ? 1 : (k <= 4 ? 4 : (k <= 8 ? 8 : (k <= 16 ? 16 : 0))); }

// The shared-memory layout of a launch in bucket kc with epilogue e (the kernel derives the same one)
tc::SmemLayout launch_layout(int n_features, int kc, tc::Epi e, int n_theta, bool rows, int row_data, bool packed = false) {
    return tc::smem_layout((n_features + 127) & ~127, tc::cfg(kc).N1, tc::cfg(kc).N2, n_theta,
                           tc::traits(e).disp ? tc::kDispWords : 0, kc, tc::row_arrays(rows, row_data), packed);
}

using LaunchFn = int (*)(const FedComm*, const GlmSegment*, const GlmParams*, const void*, const void*, int, unsigned int*,
                         int, cudaStream_t);

template <int KC, bool ROWS, tc::Epi E>
int launch(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, const void* tmaps, const void* chunks_dev,
           int n_chunks, unsigned int* work_counter, int grid, cudaStream_t stream) {
    const tc::SmemLayout L = launch_layout(prm->n_features, KC, E, comm->n_theta, ROWS, prm->row_data, prm->packed_x != 0);
    if (L.stages < 2) return -2;
    if (prm->packed_x && L.xslots < 2) return -4;
    return tc::launch_pdl(tc::fed_glm_tc_kernel<KC, ROWS, E>, grid, tc::kThreads, L.total, stream, *comm, segs_dev, *prm,
                          reinterpret_cast<const CUtensorMap*>(tmaps), reinterpret_cast<const GlmChunk*>(chunks_dev),
                          n_chunks, work_counter);
}

// The kernel's instantiations: each epilogue in every K bucket, but none that needs two columns at least
// (traits().two_columns) in KC = 1 (null).  nvcc's code for a few of them depends on the order in which they are
// instantiated, which is the order of the cases here: later epilogues go after the default.
template <tc::Epi E>
LaunchFn pick(int kc, bool rows) {
    switch (kc) {
        case 1:
            if constexpr (tc::traits(E).two_columns) return nullptr;
            else return rows ? launch<1, true, E> : launch<1, false, E>;
        case 4: return rows ? launch<4, true, E> : launch<4, false, E>;
        case 8: return rows ? launch<8, true, E> : launch<8, false, E>;
        default: return rows ? launch<16, true, E> : launch<16, false, E>;
    }
}
LaunchFn pick(tc::Epi e, int kc, bool rows) {
    using tc::Epi;
    switch (e) {
        case Epi::Hvp: return pick<Epi::Hvp>(kc, rows);
        case Epi::Softmax: return pick<Epi::Softmax>(kc, rows);
        case Epi::Ordinal: return pick<Epi::Ordinal>(kc, rows);
        case Epi::Survival: return pick<Epi::Survival>(kc, rows);
        case Epi::Dispersion: return pick<Epi::Dispersion>(kc, rows);
        default: return pick<Epi::Scalar>(kc, rows);
        case Epi::ZeroInflated: return pick<Epi::ZeroInflated>(kc, rows);
        case Epi::ZeroInflatedDisp: return pick<Epi::ZeroInflatedDisp>(kc, rows);
        case Epi::Positive: return pick<Epi::Positive>(kc, rows);
        case Epi::LocationScale: return pick<Epi::LocationScale>(kc, rows);
        case Epi::StudentT: return pick<Epi::StudentT>(kc, rows);
        case Epi::Beta: return pick<Epi::Beta>(kc, rows);
    }
}
}  // namespace

// Builds the TMA descriptors of every segment, [n_segments][4]: X ([n_rows, P] bf16, box = 64 features x 128 rows,
// 128B swizzle), then y, offset and weight ([n_rows] fp32, box = 128 rows; an absent offset / weight keeps a zeroed
// descriptor the kernel never uses), and the chunk table.  Every check comes before the first device allocation.
extern "C" int b200_glm_tc_prepare(const GlmSegment* segs_host, int n_segments, const GlmParams* prm, int sm_count,
                                   void** tmaps_dev, void** chunks_dev, int* n_chunks) {
    if (prm->n_features % 8 != 0 || prm->n_features > 384 || prm->n_features < 8) return -11;   // padded to 128s by TMA
    if (chains_bucket(prm->n_chains) == 0) return -13;
    if ((prm->ld * 2) % 16 != 0) return -14;
    const PFN_cuTensorMapEncodeTiled encode = tc::encode_tiled();
    if (!encode) return -15;
    for (int s = 0; s < n_segments; ++s) {
        const GlmSegment& g = segs_host[s];
        if (g.n_rows + tc::kTileM >= (1ll << 31)) return -18;   // row coordinates are 32-bit
        if (((uintptr_t)g.X & 15) != 0) return -16;            // TMA reads from 16-byte aligned addresses only
        if ((((uintptr_t)g.y | (uintptr_t)g.offset | (uintptr_t)g.weight) & 15) != 0) return -19;
    }
    std::vector<CUtensorMap> host((size_t)n_segments * 4);   // value-initialised: zeroed
    for (int s = 0; s < n_segments; ++s) {
        cuuint64_t dims[2] = {(cuuint64_t)prm->n_features, (cuuint64_t)segs_host[s].n_rows};
        cuuint64_t strides[1] = {(cuuint64_t)prm->ld * 2};
        cuuint32_t box[2] = {(cuuint32_t)tc::kPanel, (cuuint32_t)tc::kTileM};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&host[4 * s], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(segs_host[s].X), dims, strides,
                            box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        const float* rows[3] = {segs_host[s].y, segs_host[s].offset, segs_host[s].weight};
        for (int a = 0; a < 3 && r == CUDA_SUCCESS; ++a) {
            if (!rows[a]) continue;
            cuuint64_t rdims[1] = {(cuuint64_t)segs_host[s].n_rows};
            cuuint64_t rstrides[1] = {4};   // unused at rank 1
            cuuint32_t rbox[1] = {(cuuint32_t)tc::kTileM};
            r = encode(&host[4 * s + 1 + a], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, const_cast<float*>(rows[a]), rdims, rstrides,
                       rbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        }
        if (r != CUDA_SUCCESS) return -17;
    }
    if (*tmaps_dev) cudaFree(*tmaps_dev);
    cudaError_t e = cudaMalloc(tmaps_dev, sizeof(CUtensorMap) * host.size());
    if (e == cudaSuccess) e = cudaMemcpy(*tmaps_dev, host.data(), sizeof(CUtensorMap) * host.size(), cudaMemcpyHostToDevice);
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
extern "C" size_t b200_glm_tc_partial_row_doubles(int n_vals, int n_chains, int n_out, int n_groups, int family) {
    return tc::partial_row_doubles(n_vals, chains_bucket(n_chains), n_out > 0 ? n_out : 1, n_groups,
                                   tc::traits(tc::epilogue(family)).disp ? 1 : 0);
}

// Stages of the TMA ring the launch of this shape gets (host only; tests/test_glm_row_stream.py).  The launch
// needs at least 2.
extern "C" int b200_glm_tc_stages(int n_features, int n_chains, int n_groups, int family, int row_data) {
    const int kc = chains_bucket(n_chains);
    if (kc == 0) return 0;
    return (int)launch_layout(n_features, kc, tc::epilogue(family), 0, row_data != 0, row_data).stages;
}

// Compressed panel slots of the packed-X layout of this shape with n_theta theta words (host only): the shape can run
// packed when >= 2.
extern "C" int b200_glm_tc_packed_slots(int n_features, int n_chains, int n_groups, int family, int row_data, int n_theta) {
    const int kc = chains_bucket(n_chains);
    if (kc == 0) return 0;
    return (int)launch_layout(n_features, kc, tc::epilogue(family), n_theta, row_data != 0, row_data, true).xslots;
}

// The decoder of the packed X on the host (tests/test_glm_packed.py): one tile of `panels` kXBlock blocks, its
// footer (kXFoot bytes) and the segment's table (4 words) -> the tile's 128B-swizzled bf16 image (panels x 16 KB),
// in the order the kernel's decoders use.  Returns the exception count, or -1 for a footer that holds too many.
extern "C" int b200_glm_x12_decode_tile(const unsigned char* blocks, const int* footer, const unsigned int* tab, int panels,
                                        unsigned char* out) {
    const uint32_t t[4] = {tab[0], tab[1], tab[2], tab[3]};
    for (int pnl = 0; pnl < panels; ++pnl) {
        const unsigned char* src = blocks + (size_t)pnl * tc::kXBlock;
        for (int i = 0; i < tc::kTileM * 8; ++i) {
            uint2 lo;
            uint32_t c;
            std::memcpy(&lo, src + 8 * i, 8);
            std::memcpy(&c, src + tc::kTileM * tc::kPanel + 4 * i, 4);
            const uint4 v = tc::x12_decode8(lo, c, t);
            std::memcpy(out + (size_t)pnl * tc::kPanelBytes + tc::x12_chunk_offset(i), &v, 16);
        }
    }
    if (footer[0] < 0 || footer[0] > tc::kXMaxExceptions) return -1;
    for (int e = 0; e < footer[0]; ++e) {
        const uint32_t v = (uint32_t)footer[1 + e];
        if ((v >> 8) >= (uint32_t)panels * tc::kTileM * tc::kPanel) return -1;
        out[tc::x12_high_byte_offset(v >> 8)] = (unsigned char)(v & 0xFFu);
    }
    return footer[0];
}

extern "C" int b200_launch_glm_tc(const FedComm* comm, const GlmSegment* segs_dev, const GlmParams* prm, const void* tmaps,
                                  const void* chunks_dev, int n_chunks, unsigned int* work_counter, int grid,
                                  cudaStream_t stream) {
    const int kc = chains_bucket(prm->n_chains);
    if (kc == 0) return -1;
    const bool rows = prm->row_data != 0;   // per-row offsets / weights somewhere: the instantiation that reads them
    const LaunchFn fn = pick(tc::epilogue(prm->family), kc, rows);
    if (!fn) return -3;
    return fn(comm, segs_dev, prm, tmaps, chunks_dev, n_chunks, work_counter, grid, stream);
}
