// Federated ODE parameter estimation: [timepoints, theta] -> trajectories -> LL and dLL/dtheta.
//
// Workload named in BASELINE.json ("federated ODE parameter estimation ... 4 shards
// on 4 GPUs"); the reference only describes it in prose (README.md:39-52: the
// federated function is an ODE solve whose data never leaves the node).  Model: Lotka-Volterra
//     u' = alpha u - beta u v ,  v' = delta u v - gamma v ,  theta = (alpha, beta, gamma, delta)
// with forward sensitivities S = d(u,v)/dtheta integrated alongside (10 coupled ODEs), classic
// RK4, one thread per observed series.  No tensor-core work here: the op is latency/ALU bound
// and the fused broadcast -> solve -> reduce path (fed_comm.cuh) is what matters.
#include "fed_comm.cuh"
#include "models.h"

namespace {

struct State {
    float u, v;
    float su[4], sv[4];
};

__device__ __forceinline__ void rhs(const State& s, const float th[4], State& d) {
    const float a = th[0], b = th[1], g = th[2], dl = th[3];
    const float uv = s.u * s.v;
    d.u = a * s.u - b * uv;
    d.v = dl * uv - g * s.v;
    // Jacobian
    const float fuu = a - b * s.v, fuv = -b * s.u;
    const float fvu = dl * s.v, fvv = dl * s.u - g;
    // explicit parameter derivatives
    const float pu[4] = {s.u, -uv, 0.f, 0.f};
    const float pv[4] = {0.f, 0.f, -s.v, uv};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        d.su[k] = fuu * s.su[k] + fuv * s.sv[k] + pu[k];
        d.sv[k] = fvu * s.su[k] + fvv * s.sv[k] + pv[k];
    }
}

__device__ __forceinline__ State axpy(const State& s, float h, const State& d) {
    State r;
    r.u = fmaf(h, d.u, s.u);
    r.v = fmaf(h, d.v, s.v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        r.su[k] = fmaf(h, d.su[k], s.su[k]);
        r.sv[k] = fmaf(h, d.sv[k], s.sv[k]);
    }
    return r;
}

__device__ __forceinline__ void rk4_step(State& s, const float th[4], float h) {
    State k1, k2, k3, k4;
    rhs(s, th, k1);
    rhs(axpy(s, 0.5f * h, k1), th, k2);
    rhs(axpy(s, 0.5f * h, k2), th, k3);
    rhs(axpy(s, h, k3), th, k4);
    const float h6 = h * (1.f / 6.f);
    s.u += h6 * (k1.u + 2.f * k2.u + 2.f * k3.u + k4.u);
    s.v += h6 * (k1.v + 2.f * k2.v + 2.f * k3.v + k4.v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        s.su[k] += h6 * (k1.su[k] + 2.f * k2.su[k] + 2.f * k3.su[k] + k4.su[k]);
        s.sv[k] += h6 * (k1.sv[k] + 2.f * k2.sv[k] + 2.f * k3.sv[k] + k4.sv[k]);
    }
}

constexpr int kMaxTheta = 1024;   // floats of theta staged in shared memory (nodes x 4)

// theta holds one (alpha, beta, gamma, delta) per node and the result one [LL, dLL/dtheta] block per node:
// every shard names its own (theta_offset, out_offset), so the client may give each node its own parameters
// and weight / sum the node results itself (the reference's one-Op-per-node pattern), still in ONE launch.
__global__ void __launch_bounds__(128) fed_ode_kernel(FedComm comm, const OdeShard* __restrict__ shards, int n_shards) {
    __shared__ float theta[kMaxTheta];
    __shared__ double red[32];
    fed::Prologue pro = fed::prologue(comm, theta);
    if (!pro.stop && !pro.timed_out) {
        double* out = comm.cta_partials + (size_t)blockIdx.x * comm.n_vals;
        for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) out[i] = 0.0;
        __syncthreads();
        for (int sidx = 0; sidx < n_shards; ++sidx) {
            const OdeShard sh = shards[sidx];
            const float th[4] = {theta[sh.theta_offset], theta[sh.theta_offset + 1], theta[sh.theta_offset + 2],
                                 theta[sh.theta_offset + 3]};
            double acc[5] = {0, 0, 0, 0, 0};  // LL, dLL/dtheta[4]
            const float inv_var = 1.f / (sh.sigma * sh.sigma);
            const float log_norm = -__logf(sh.sigma) - 0.918938533204672742f;
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < sh.n_series; i += gridDim.x * blockDim.x) {
                State s;
                s.u = sh.y0[i];
                s.v = sh.y0[sh.n_series + i];
#pragma unroll
                for (int k = 0; k < 4; ++k) s.su[k] = s.sv[k] = 0.f;
                float t_prev = 0.f;
                float ll = 0.f, g[4] = {0.f, 0.f, 0.f, 0.f};
                for (int j = 0; j < sh.n_t; ++j) {
                    const float t_next = sh.t[j];
                    const float h = (t_next - t_prev) / (float)sh.substeps;
                    for (int q = 0; q < sh.substeps; ++q) rk4_step(s, th, h);
                    t_prev = t_next;
                    const float ou = sh.y_obs[((size_t)j * 2 + 0) * sh.n_series + i];
                    const float ov = sh.y_obs[((size_t)j * 2 + 1) * sh.n_series + i];
                    const float ru = ou - s.u, rv = ov - s.v;
                    ll += -0.5f * (ru * ru + rv * rv) * inv_var + 2.f * log_norm;
#pragma unroll
                    for (int k = 0; k < 4; ++k) g[k] += (ru * s.su[k] + rv * s.sv[k]) * inv_var;
                }
                acc[0] += (double)ll;
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[1 + k] += (double)g[k];
            }
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const double v = fed::block_sum(acc[k], red);
                if (threadIdx.x == 0) out[sh.out_offset + k] += v;
            }
        }
    }
    fed::epilogue(comm, pro, 0ull);
}

}  // namespace

extern "C" int b200_launch_ode(const FedComm* comm, const OdeShard* shards_dev, int n_shards, int grid,
                               cudaStream_t stream) {
    if (comm->n_theta % 4 != 0 || comm->n_theta > kMaxTheta || comm->n_vals % 5 != 0) return -1;
    fed_ode_kernel<<<grid, 128, 0, stream>>>(*comm, shards_dev, n_shards);
    return (int)cudaGetLastError();
}
