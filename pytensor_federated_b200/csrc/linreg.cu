// Federated Gaussian linear regression: per-shard  LL, dLL/d(intercept), dLL/d(slope).
//
// Maths of the reference's only shipped model (demo_node.py:31-43):
//   pred = a + b*x ;  LL = sum log N(y | pred, sigma)
//   dLL/da = sum (y-pred)/sigma^2 ;  dLL/db = sum (y-pred)*x/sigma^2
// The reference evaluates this in a PyTensor-compiled CPU function behind gRPC; here it
// is one fused broadcast->compute->reduce kernel (see fed_comm.cuh).  Each shard has its
// own (intercept, slope) pair in theta so that hierarchical models
// (demo_model.py:28-36: per-group intercepts, shared slope) evaluate all
// of their remote calls in ONE launch.  Everything is fp64: the reference returns float64
// and its users compare against NumPy at ~1e-12.
#include "fed_comm.cuh"
#include "models.h"

namespace {

template <typename T>
__global__ void __launch_bounds__(256) fed_linreg_kernel(FedComm comm, const LinregShard* __restrict__ shards,
                                                          int n_shards, int small_mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* theta_words = reinterpret_cast<float*>(smem_raw);                       // n_theta words
    double* red = reinterpret_cast<double*>(smem_raw + ((comm.n_theta * 4 + 15) & ~15));  // 32 doubles

    fed::Prologue pro = fed::prologue(comm, theta_words);
    unsigned long long status = 0;
    if (!pro.stop && !pro.timed_out) {
        const double* theta = reinterpret_cast<const double*>(theta_words);
        double* out = comm.cta_partials + (size_t)blockIdx.x * comm.n_vals;
        // entries of shards that live on other nodes must read as zero in the cross-node sum
        for (int i = threadIdx.x; i < comm.n_vals; i += blockDim.x) out[i] = 0.0;
        __syncthreads();
        if (small_mode) {
            // tiny shards (the reference's demo: 10 rows per node): one warp per shard, shuffle
            // reductions only — no block-wide barriers on the latency path
            const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
            for (int s = warp; s < n_shards; s += n_warps) {
                const LinregShard sh = shards[s];
                const double a = theta[sh.theta_offset];
                const double b = theta[sh.theta_offset + 1];
                const T* __restrict__ x = reinterpret_cast<const T*>(sh.x);
                const T* __restrict__ y = reinterpret_cast<const T*>(sh.y);
                double s_rr = 0.0, s_r = 0.0, s_rx = 0.0;
                for (long long i = lane; i < sh.n; i += 32) {
                    const double xi = (double)x[i];
                    const double r = (double)y[i] - (a + b * xi);
                    s_rr += r * r;
                    s_r += r;
                    s_rx += r * xi;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    s_rr += __shfl_xor_sync(0xffffffffu, s_rr, o);
                    s_r += __shfl_xor_sync(0xffffffffu, s_r, o);
                    s_rx += __shfl_xor_sync(0xffffffffu, s_rx, o);
                }
                if (lane == 0) {
                    const double inv_var = 1.0 / (sh.sigma * sh.sigma);
                    const double log_norm = -log(sh.sigma) - 0.91893853320467274178;
                    const int gs = sh.theta_offset / 2;
                    out[gs * 3 + 0] = -0.5 * s_rr * inv_var + (double)sh.n * log_norm;
                    out[gs * 3 + 1] = s_r * inv_var;
                    out[gs * 3 + 2] = s_rx * inv_var;
                }
            }
        } else
        for (int s = 0; s < n_shards; ++s) {
            const LinregShard sh = shards[s];
            const double a = theta[sh.theta_offset];
            const double b = theta[sh.theta_offset + 1];
            const T* __restrict__ x = reinterpret_cast<const T*>(sh.x);
            const T* __restrict__ y = reinterpret_cast<const T*>(sh.y);
            double s_rr = 0.0, s_r = 0.0, s_rx = 0.0;
            for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < sh.n;
                 i += (long long)gridDim.x * blockDim.x) {
                const double xi = (double)x[i];
                const double r = (double)y[i] - (a + b * xi);
                s_rr += r * r;
                s_r += r;
                s_rx += r * xi;
            }
            s_rr = fed::block_sum(s_rr, red);
            s_r = fed::block_sum(s_r, red);
            s_rx = fed::block_sum(s_rx, red);
            if (threadIdx.x == 0) {
                const double inv_var = 1.0 / (sh.sigma * sh.sigma);
                // rows handled by this CTA (for the constant term)
                long long n_here = 0;
                {
                    const long long stride = (long long)gridDim.x * blockDim.x;
                    const long long first = (long long)blockIdx.x * blockDim.x;
                    if (sh.n > first) {
                        const long long full = (sh.n - first) / stride;       // complete strides
                        const long long rem = (sh.n - first) - full * stride;  // leftover rows in the last stride
                        n_here = full * blockDim.x + (rem < (long long)blockDim.x ? rem : (long long)blockDim.x);
                    }
                }
                const double log_norm = -log(sh.sigma) - 0.91893853320467274178;  // -log(sigma*sqrt(2*pi))
                const int gs = sh.theta_offset / 2;  // global shard index
                out[gs * 3 + 0] = -0.5 * s_rr * inv_var + (double)n_here * log_norm;
                out[gs * 3 + 1] = s_r * inv_var;
                out[gs * 3 + 2] = s_rx * inv_var;
            }
        }
    }
    fed::epilogue(comm, pro, status);
}

}  // namespace

extern "C" int b200_launch_linreg(const FedComm* comm, const LinregShard* shards_dev, int n_shards, int dtype_is_f64,
                                  int grid, cudaStream_t stream) {
    // theta (16 bytes per shard of the federation) lives in dynamic shared memory: from 3056 shards on, it and the
    // kernel's static variables (< 256 bytes) need more than the default 48 KB, which a launch gets only after
    // opting in, up to 227 KB (LinregShards.MAX_SHARDS_TOTAL).  Smaller models skip the call and launch as before.
    const size_t smem = ((comm->n_theta * 4 + 15) & ~15) + 32 * sizeof(double);
    const int small_mode = grid < 0 ? 1 : 0;  // negative grid = "one CTA, warp per shard"
    if (grid < 0) grid = 1;
    if (smem > 48 * 1024 - 256) {
        const cudaError_t err =
            dtype_is_f64 ? cudaFuncSetAttribute(fed_linreg_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                         : cudaFuncSetAttribute(fed_linreg_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return (int)err;
    }
    if (dtype_is_f64)
        fed_linreg_kernel<double><<<grid, 256, smem, stream>>>(*comm, shards_dev, n_shards, small_mode);
    else
        fed_linreg_kernel<float><<<grid, 256, smem, stream>>>(*comm, shards_dev, n_shards, small_mode);
    return (int)cudaGetLastError();
}
