// Federated ODE parameter estimation for a USER-SUPPLIED right-hand side.
//
// The reference's premise is that the federated function is arbitrary — its README describes "an ODE solve
// whose data never leaves the node" (README.md:39-52).  csrc/ode.cu hard-codes one system
// (Lotka-Volterra with hand-written sensitivities); this file is the general case: the user writes ONLY the
// right-hand side, once, as a snippet of CUDA C over a scalar type `T`
//
//     dy[0] = th[0] * y[0] - th[1] * y[0] * y[1];          // inputs: y[NS], th[NP], t;  output: dy[NS]
//     dy[1] = th[3] * y[0] * y[1] - th[2] * y[1];
//
// and the kernel integrates it with classic RK4 on FORWARD-MODE DUAL NUMBERS (value + NP partial derivatives,
// operators and elementary functions below), which yields the trajectory and d(trajectory)/d(theta) of the
// same discrete scheme — exactly what integrating the sensitivity equations alongside would give, without
// asking the user for Jacobians.  One thread per observed series; Gaussian observation noise on every state;
// broadcast -> solve -> reduce through fed_comm.cuh like every other model.
//
// Compiled per system by models/ode.py (nvcc, cached by content hash) with
//   -DB200FED_ODE_NS=<states> -DB200FED_ODE_NP=<parameters> -DB200FED_ODE_RHS=<snippet>
// Without those macros this file builds the Lotka-Volterra instance (used by the tests as a cross-check of ode.cu).
#include "fed_comm.cuh"
#include "models.h"

#ifndef B200FED_ODE_NS
#define B200FED_ODE_NS 2
#define B200FED_ODE_NP 4
#define B200FED_ODE_RHS                          \
    dy[0] = th[0] * y[0] - th[1] * y[0] * y[1]; \
    dy[1] = th[3] * y[0] * y[1] - th[2] * y[1];
#endif
#ifndef B200FED_ODE_ENTRY
#define B200FED_ODE_ENTRY b200_launch_ode_generic
#endif

namespace odeg {

constexpr int NS = B200FED_ODE_NS;
constexpr int NP = B200FED_ODE_NP;
constexpr int kMaxTheta = 1024;   // floats of theta staged in shared memory (nodes x NP)

// ---- forward-mode dual number: v + sum_k d[k] eps_k ------------------------------------------------------
struct Dual {
    float v;
    float d[NP];
};
__device__ __forceinline__ Dual make_const(float c) {
    Dual r;
    r.v = c;
#pragma unroll
    for (int k = 0; k < NP; ++k) r.d[k] = 0.f;
    return r;
}
// r = f(a) with derivative factor fa: r.d = fa * a.d
__device__ __forceinline__ Dual chain1(float value, float fa, const Dual& a) {
    Dual r;
    r.v = value;
#pragma unroll
    for (int k = 0; k < NP; ++k) r.d[k] = fa * a.d[k];
    return r;
}
__device__ __forceinline__ Dual chain2(float value, float fa, const Dual& a, float fb, const Dual& b) {
    Dual r;
    r.v = value;
#pragma unroll
    for (int k = 0; k < NP; ++k) r.d[k] = fmaf(fa, a.d[k], fb * b.d[k]);
    return r;
}
__device__ __forceinline__ Dual operator+(const Dual& a, const Dual& b) { return chain2(a.v + b.v, 1.f, a, 1.f, b); }
__device__ __forceinline__ Dual operator-(const Dual& a, const Dual& b) { return chain2(a.v - b.v, 1.f, a, -1.f, b); }
__device__ __forceinline__ Dual operator*(const Dual& a, const Dual& b) { return chain2(a.v * b.v, b.v, a, a.v, b); }
__device__ __forceinline__ Dual operator/(const Dual& a, const Dual& b) {
    const float inv = 1.f / b.v;
    return chain2(a.v * inv, inv, a, -a.v * inv * inv, b);
}
__device__ __forceinline__ Dual operator-(const Dual& a) { return chain1(-a.v, -1.f, a); }
__device__ __forceinline__ Dual operator+(const Dual& a, float c) { return chain1(a.v + c, 1.f, a); }
__device__ __forceinline__ Dual operator+(float c, const Dual& a) { return chain1(a.v + c, 1.f, a); }
__device__ __forceinline__ Dual operator-(const Dual& a, float c) { return chain1(a.v - c, 1.f, a); }
__device__ __forceinline__ Dual operator-(float c, const Dual& a) { return chain1(c - a.v, -1.f, a); }
__device__ __forceinline__ Dual operator*(const Dual& a, float c) { return chain1(a.v * c, c, a); }
__device__ __forceinline__ Dual operator*(float c, const Dual& a) { return chain1(a.v * c, c, a); }
__device__ __forceinline__ Dual operator/(const Dual& a, float c) { return chain1(a.v / c, 1.f / c, a); }
__device__ __forceinline__ Dual operator/(float c, const Dual& a) { return chain1(c / a.v, -c / (a.v * a.v), a); }
__device__ __forceinline__ Dual exp(const Dual& a) { const float e = expf(a.v); return chain1(e, e, a); }
__device__ __forceinline__ Dual log(const Dual& a) { return chain1(logf(a.v), 1.f / a.v, a); }
__device__ __forceinline__ Dual sqrt(const Dual& a) { const float s = sqrtf(a.v); return chain1(s, 0.5f / s, a); }
__device__ __forceinline__ Dual sin(const Dual& a) { return chain1(sinf(a.v), cosf(a.v), a); }
__device__ __forceinline__ Dual cos(const Dual& a) { return chain1(cosf(a.v), -sinf(a.v), a); }
__device__ __forceinline__ Dual tanh(const Dual& a) { const float t = tanhf(a.v); return chain1(t, 1.f - t * t, a); }
__device__ __forceinline__ Dual pow(const Dual& a, float p) { return chain1(powf(a.v, p), p * powf(a.v, p - 1.f), a); }
__device__ __forceinline__ Dual square(const Dual& a) { return chain1(a.v * a.v, 2.f * a.v, a); }
// plain-float overloads so that a snippet may call the same names on constants
__device__ __forceinline__ float square(float a) { return a * a; }

// The user's right-hand side.  `T` is Dual here; the snippet must not name the type.
template <typename T>
__device__ __forceinline__ void rhs(const T (&y)[NS], const T (&th)[NP], float t, T (&dy)[NS]) {
    (void)t;
    B200FED_ODE_RHS
}

struct State {
    Dual y[NS];
};
__device__ __forceinline__ State axpy(const State& s, float h, const State& d) {
    State r;
#pragma unroll
    for (int i = 0; i < NS; ++i) {
        r.y[i].v = fmaf(h, d.y[i].v, s.y[i].v);
#pragma unroll
        for (int k = 0; k < NP; ++k) r.y[i].d[k] = fmaf(h, d.y[i].d[k], s.y[i].d[k]);
    }
    return r;
}
__device__ __forceinline__ void rk4_step(State& s, const Dual (&th)[NP], float t, float h) {
    State k1, k2, k3, k4;
    rhs<Dual>(s.y, th, t, k1.y);
    rhs<Dual>(axpy(s, 0.5f * h, k1).y, th, t + 0.5f * h, k2.y);
    rhs<Dual>(axpy(s, 0.5f * h, k2).y, th, t + 0.5f * h, k3.y);
    rhs<Dual>(axpy(s, h, k3).y, th, t + h, k4.y);
    const float h6 = h * (1.f / 6.f);
#pragma unroll
    for (int i = 0; i < NS; ++i) {
        s.y[i].v += h6 * (k1.y[i].v + 2.f * k2.y[i].v + 2.f * k3.y[i].v + k4.y[i].v);
#pragma unroll
        for (int k = 0; k < NP; ++k)
            s.y[i].d[k] += h6 * (k1.y[i].d[k] + 2.f * k2.y[i].d[k] + 2.f * k3.y[i].d[k] + k4.y[i].d[k]);
    }
}

// Data layout (models/ode.py): y0 [NS, n_series], y_obs [n_t, NS, n_series] (series index fastest).
__global__ void __launch_bounds__(128) fed_ode_generic_kernel(FedComm comm, const OdeShard* __restrict__ shards, int n_shards) {
    __shared__ float theta[kMaxTheta];
    __shared__ double red[32];
    fed::Prologue pro = fed::prologue(comm, theta);
    if (!pro.stop && !pro.timed_out) {
        double* out = comm.cta_partials + (size_t)blockIdx.x * comm.n_vals;
        for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) out[i] = 0.0;
        __syncthreads();
        for (int sidx = 0; sidx < n_shards; ++sidx) {
            const OdeShard sh = shards[sidx];
            // per-node parameters and result block (see csrc/ode.cu)
            Dual th[NP];
#pragma unroll
            for (int k = 0; k < NP; ++k) {
                th[k] = make_const(theta[sh.theta_offset + k]);
                th[k].d[k] = 1.f;
            }
            double acc[1 + NP];
#pragma unroll
            for (int k = 0; k <= NP; ++k) acc[k] = 0.0;
            const float inv_var = 1.f / (sh.sigma * sh.sigma);
            const float log_norm = -__logf(sh.sigma) - 0.918938533204672742f;
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < sh.n_series; i += gridDim.x * blockDim.x) {
                State s;
#pragma unroll
                for (int c = 0; c < NS; ++c) s.y[c] = make_const(sh.y0[(size_t)c * sh.n_series + i]);
                float t_prev = 0.f;
                float ll = 0.f, g[NP];
#pragma unroll
                for (int k = 0; k < NP; ++k) g[k] = 0.f;
                for (int j = 0; j < sh.n_t; ++j) {
                    const float t_next = sh.t[j];
                    const float h = (t_next - t_prev) / (float)sh.substeps;
                    for (int q = 0; q < sh.substeps; ++q) rk4_step(s, th, t_prev + (float)q * h, h);
                    t_prev = t_next;
#pragma unroll
                    for (int c = 0; c < NS; ++c) {
                        const float r = sh.y_obs[((size_t)j * NS + c) * sh.n_series + i] - s.y[c].v;
                        ll += -0.5f * r * r * inv_var + log_norm;
#pragma unroll
                        for (int k = 0; k < NP; ++k) g[k] += r * s.y[c].d[k] * inv_var;
                    }
                }
                acc[0] += (double)ll;
#pragma unroll
                for (int k = 0; k < NP; ++k) acc[1 + k] += (double)g[k];
            }
#pragma unroll
            for (int k = 0; k <= NP; ++k) {
                const double v = fed::block_sum(acc[k], red);
                if (threadIdx.x == 0) out[sh.out_offset + k] += v;
            }
        }
    }
    fed::epilogue(comm, pro, 0ull);
}

}  // namespace odeg

extern "C" int B200FED_ODE_ENTRY(const FedComm* comm, const OdeShard* shards_dev, int n_shards, int grid, cudaStream_t stream) {
    if (comm->n_theta % odeg::NP != 0 || comm->n_theta > odeg::kMaxTheta || comm->n_vals % (1 + odeg::NP) != 0) return -1;
    odeg::fed_ode_generic_kernel<<<grid, 128, 0, stream>>>(*comm, shards_dev, n_shards);
    return (int)cudaGetLastError();
}
extern "C" int b200_ode_generic_dims(int* ns, int* np) {
    *ns = odeg::NS;
    *np = odeg::NP;
    return 0;
}
