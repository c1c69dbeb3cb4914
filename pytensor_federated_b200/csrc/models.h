// Plain-old-data descriptors shared between the host runtime and the kernels.
#pragma once
#include <cstdint>

struct LinregShard {
    const void* x;        // [n] float64 or float32
    const void* y;        // [n]
    long long n;
    double sigma;
    int theta_offset;     // index (in doubles) of this shard's (intercept, slope) pair in theta
    int _pad;
};

// One contiguous block of rows of a generalised linear model ("shard" / "group").
struct GlmSegment {
    const void* X;        // [n_rows, ld] row-major; bf16 (or fp8 e4m3 for the block-scaled kernel)
    const float* y;       // [n_rows] response (0/1 for logistic)
    const void* scales;   // fp8 only: per-(row, 32-feature block) ue8m0 scales, else null
    const float* offset;  // [n_rows] known part of eta added after the intercept, or null (no offset)
    const float* weight;  // [n_rows] observation weights (>= 0; 0 masks the row), or null (weight 1)
    long long n_rows;
    long long first_tile; // prefix sum over segments of ceil(n_rows / tile_rows)
    int group;            // which intercept this segment uses
    int out_group;        // which output block this segment's [LL, grads] go to (0 unless per-node outputs are kept)
    // bf16 tensor-core kernel, GlmParams::packed_x: X as a lossless 12-bit code (tc::x12_decode8), one 12 KB block per
    // (128-row tile, 64-feature panel) in tile-major order, a 256-byte exception footer per tile, and the segment's
    // 16-entry table of high bytes (entry 4 q + b in byte b of xtab[q])
    const void* xpack;
    const void* xfoot;
    unsigned int xtab[4];
};

struct GlmParams {
    int n_segments;
    int n_features;       // P
    int ld;               // row stride of X in elements
    int n_groups;         // G intercepts; theta = [intercept[G], beta[P]] per chain ([.., log_dispersion] where glm_family().dispersion)
    int n_chains;         // K parameter vectors evaluated per launch (theta is [K][G+P], [K][G+P+1] with a dispersion word)
    int family;           // a GlmFamilyCode, or kGlmHvp | (0, 1 or 2)
    long long total_tiles;
    int n_out;            // output blocks: 1 = everything summed; > 1 = one [K][1+G+P] block per node (tensor-core kernel)
    int early_loads;      // tensor-core kernels: claim + load the first tiles before theta arrives (B200FED_NO_EARLY_LOADS=1: off)
    int row_data;         // kGlmRowOffsets | kGlmRowWeights when any segment has them: selects the kernel instantiation
    int n_classes;        // C: multinomial classes or ordinal categories (GlmFamily::columns), else 1.  Theta row v holds
                          // column v: (intercept[:, c], beta[:, c]) of class c, (intercept - c_j, beta) of cutpoint j
    int packed_x;         // bf16 tensor-core kernel: X is read from GlmSegment::xpack / xfoot (B200FED_NO_PACKED_X=1: never)
};

constexpr int kGlmRowOffsets = 1;
constexpr int kGlmRowWeights = 2;
// Flag bit on GlmParams::family: the launch evaluates pairs of columns, column 2k the parameters theta_k and column
// 2k + 1 a direction v_k, whose output block is [0, (H v)_intercept[G], (H v)_beta[P]] with H the Hessian of LL at
// theta_k.  Only the bf16 tensor-core kernel takes it (families 0 to 2, an even n_chains); the runtime refuses it
// for every other kernel.
constexpr int kGlmHvp = 16;

// GlmParams::family (models/glm.py FAMILIES holds the same codes)
enum GlmFamilyCode : int {
    kGlmLogistic = 0,        // Bernoulli, logit link
    kGlmPoisson = 1,         // log link
    kGlmGaussian = 2,        // identity link, unit variance
    kGlmMultinomial = 3,     // softmax over n_classes columns
    kGlmGaussianScale = 4,   // Gaussian with unknown scale, log_dispersion = log sigma
    kGlmNegBinomial = 5,     // NB2, log link, log_dispersion = log alpha
    kGlmOrdinal = 6,         // cumulative logit over n_classes categories, one column per cutpoint
    kGlmWeibull = 7,         // right-censored survival (AFT), log_dispersion = log sigma,
    kGlmLogNormal = 8,       //   y = +t for an event, -t for a censored row
    kGlmZeroInflatedPoisson = 9,       // zero-inflated counts: pair p is column 2p (count eta) and 2p + 1 (zero logit
    kGlmZeroInflatedNegBinomial = 10,  //   zeta); family 10 adds NB2's log_dispersion = log alpha
    kGlmGamma = 11,          // positive responses, log link to the mean, log_dispersion = log shape (nu, lambda):
    kGlmInverseGaussian = 12,  //   Var(y) = mu^2 / nu (gamma), mu^3 / lambda (inverse Gaussian)
    kGlmGaussianLocationScale = 13,  // location-scale: pair p is column 2p (mean mu, identity link) and 2p + 1
    kGlmStudentT = 14,               //   (log sigma); family 14 adds log_dispersion = log nu
    kGlmBeta = 15,           // proportions in (0, 1), logit link to the mean, log_dispersion = log precision phi:
                             //   Var(y) = mu (1 - mu) / (1 + phi)
};

// How a family's columns make up n_chains: one per chain, one per chain and class (column k C + c is class c of chain
// k), one per chain and cutpoint (column k (C - 1) + j is cutpoint j of chain k), for C = n_classes, or two per chain
// (column 2k and 2k + 1: the zero-inflated families' count and zero predictors, the location-scale families' mean and
// log sigma)
enum class GlmColumns { kOne, kPerClass, kPerCutpoint, kPair };

// What the runtime and the bf16 tensor-core kernel need to know about a family code.
struct GlmFamily {
    const char* name;        // as in models/glm.py
    bool tc_only;            // runs on the bf16 tensor-core kernel only
    bool dispersion;         // theta rows and output blocks end in a log_dispersion word: [LL, gi[G], g[P], dLL/dlog_dispersion]
    GlmColumns columns;
    int min_classes, max_classes;
    bool offsets;            // takes per-row offsets
};
constexpr GlmFamily glm_family(int code) {
    switch (code) {
        case kGlmMultinomial: return {"multinomial", true, false, GlmColumns::kPerClass, 2, 16, false};
        case kGlmGaussianScale: return {"gaussian_scale", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmNegBinomial: return {"negative_binomial", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmOrdinal: return {"ordinal", true, false, GlmColumns::kPerCutpoint, 2, 17, true};
        case kGlmWeibull: return {"weibull", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmLogNormal: return {"lognormal", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmZeroInflatedPoisson: return {"zero_inflated_poisson", true, false, GlmColumns::kPair, 1, 1, true};
        case kGlmZeroInflatedNegBinomial:
            return {"zero_inflated_negative_binomial", true, true, GlmColumns::kPair, 1, 1, true};
        case kGlmGamma: return {"gamma", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmInverseGaussian: return {"inverse_gaussian", true, true, GlmColumns::kOne, 1, 1, true};
        case kGlmGaussianLocationScale:
            return {"gaussian_location_scale", true, false, GlmColumns::kPair, 1, 1, true};
        case kGlmStudentT: return {"student_t", true, true, GlmColumns::kPair, 1, 1, true};
        case kGlmBeta: return {"beta", true, true, GlmColumns::kOne, 1, 1, true};
        default: return {"", false, false, GlmColumns::kOne, 1, 1, true};   // 0 to 2: every GLM kernel
    }
}

// Unit of work of the dynamically scheduled tensor-core GLM kernel: n_tiles consecutive 128-row tiles of one
// segment starting at tile first_tile (n_tiles is even; the last one may lie past the segment's rows).
struct GlmChunk {
    int seg;
    int first_tile;
    int n_tiles;
    int _pad;
};

// Lotka-Volterra parameter estimation: every series i starts from its own (known) state
// y0[:, i] and is observed at the shared time grid t[0..n_t).
struct OdeShard {
    const float* t;       // [n_t] observation times (ascending, t[0] > 0; integration starts at 0)
    const float* y0;      // [2, n_series]   initial prey / predator densities
    const float* y_obs;   // [n_t, 2, n_series] noisy observations (series index fastest)
    int n_series;
    int n_t;
    float sigma;          // observation noise (Gaussian)
    int substeps;         // RK4 steps between consecutive observation times
    int theta_offset;     // first float of this shard's parameter vector in theta (per-node parameters)
    int out_offset;       // first double of this shard's [LL, dLL/dtheta] block in the result
};
