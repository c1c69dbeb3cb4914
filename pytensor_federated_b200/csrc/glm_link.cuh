// Per-row likelihood of GLM families 0 to 2, shared by every GLM kernel: the SIMT, general-shape and tensor-core
// kernels are tested against each other bit for bit, so they evaluate these very expressions.
#pragma once
#include <cuda_runtime.h>

__device__ __forceinline__ void link_loglik(int family, float y, float eta, float& ll, float& r) {
    if (family == 0) {  // Bernoulli / logit
        const float e = __expf(-fabsf(eta));
        const float sp = fmaxf(eta, 0.f) + __logf(1.f + e);       // softplus(eta)
        const float inv = __fdividef(1.f, 1.f + e);
        const float p = eta >= 0.f ? inv : e * inv;               // sigmoid(eta)
        ll = y * eta - sp;
        r = y - p;
    } else if (family == 1) {  // Poisson / log (constant -lgamma(y+1) omitted)
        const float mu = __expf(eta);
        ll = y * eta - mu;
        r = y - mu;
    } else {  // Gaussian / identity, unit variance
        const float d = y - eta;
        ll = -0.5f * d * d - 0.918938533204672742f;
        r = d;
    }
}

// h = d2ll / deta2 of families 0 to 2 at eta (the Hessian-vector product's per-row weight): logistic -mu (1 - mu) =
// -e / (1 + e)^2 with e = exp(-|eta|), from an accurate expf so that h keeps its relative accuracy in both tails;
// Poisson -mu, the very __expf(eta) that link_loglik's residual uses; Gaussian -1.
__device__ __forceinline__ float link_curvature(int family, float eta) {
    if (family == 0) {
        const float e = expf(-fabsf(eta));
        const float d = 1.f + e;
        return -e / (d * d);
    }
    return family == 1 ? -__expf(eta) : -1.f;
}

// x *= wt for a row's value and its observation weight, rounded on its own (no FMA contraction, so w = 1 gives the bits
// of the unweighted model); a zero weight gives exactly 0, so a masked row's non-finite y or offset never reaches a sum.
__device__ __forceinline__ void apply_weight(float wt, float& x) { x = wt == 0.f ? 0.f : __fmul_rn(wt, x); }
