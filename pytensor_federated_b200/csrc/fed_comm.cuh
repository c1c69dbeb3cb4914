// Device-side federation protocol shared by every model kernel (sm_90a).
//
// One evaluation ("epoch") of a federated log-likelihood is ONE kernel per GPU:
//
//   prologue   rank 0 ("root", the client's GPU) reads theta from host-mapped
//              pinned memory and stores it into every node's theta mailbox over
//              NVLink (multimem.st through the NVSwitch multicast object when one
//              exists, otherwise one P2P store per peer), then releases an epoch
//              flag per node.  Every CTA of every node acquires its local flag.
//   compute    model specific (linreg / GLM / ODE ...), per-CTA partials.
//   epilogue   last CTA of each node sums the CTA partials in a fixed order and
//              stores the node's [LL, dLL/dtheta] into the root's slot array over
//              NVLink + releases a slot flag.  The root's last CTA acquires all
//              slot flags, sums the nodes in rank order (deterministic), and
//              writes the result + a completion flag into host-mapped memory.
//
// This replaces the reference's per-evaluation path of
//   npproto encode -> HTTP/2 send -> decode -> compute -> encode -> recv -> decode
// (pytensor_federated/service.py:150-158, :45-72) and the
// client-side graph sum over nodes, with zero host involvement on the nodes.
//
// Memory-model notes: data is written with weak stores, then
// __threadfence_system(); the flag is written with st.release.sys and read with
// ld.acquire.sys (the acquire invalidates the SM's L1, and mailbox data is
// re-read with ld.cg on top of that).  Epoch tags make stale flags detectable; every
// spin is bounded by %globaltimer so a dead peer yields an error code instead
// of a hung GPU.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#define B200FED_MAX_WORLD 8

// status bits OR-ed into the completion flag's upper byte
#define B200FED_STATUS_SHIFT 56
#define B200FED_EPOCH_MASK 0x00FFFFFFFFFFFFFFull
#define B200FED_ERR_THETA_TIMEOUT 1ull
#define B200FED_ERR_PEER_TIMEOUT 2ull
#define B200FED_ERR_PIPELINE 4ull      // a tensor-core kernel's mbarrier pipeline stalled (tc_common.cuh)
#define B200FED_STOP_EPOCH 0x00FFFFFFFFFFFFFFull

struct FedComm {
    int rank;                 // 0 = root (client GPU)
    int world;                // number of nodes (GPUs)
    int n_theta;              // floats in the theta mailbox
    int n_vals;               // doubles per node partial: [LL, grads...]
    unsigned long long epoch; // this launch's epoch (root: passed by host; peer: see epoch_counter)
    unsigned long long timeout_ns;

    // --- root only ---------------------------------------------------------
    const float* theta_src;                        // host-mapped pinned (or device) theta
    float* peer_theta[B200FED_MAX_WORLD];          // every node's mailbox (incl. own)
    unsigned long long* peer_flag[B200FED_MAX_WORLD];
    float* mc_theta;                               // multicast alias of the mailbox (or null)
    unsigned long long* mc_flag;                   // multicast alias of the flag (or null)
    double* host_result;                           // host-mapped [n_vals]
    unsigned long long* host_flag;                 // host-mapped completion flag

    // --- every node ----------------------------------------------------------
    float* theta_local;                            // own mailbox
    unsigned long long* flag_local;                // own epoch flag
    double* root_slots;                            // root's slot array [world][n_vals]   (peer memory)
    unsigned long long* root_slot_flags;           // root's slot flags [world]             (peer memory)
    double* cta_partials;                          // local scratch [grid][n_vals]
    double* group_partials;                        // local scratch of the two-level reduction [grid/16][n_vals] (x2 for pairs)
    unsigned int* ticket;                          // [0]: groups finished; [1 + g]: CTAs of group g finished
    unsigned long long* epoch_counter;             // peers: device-resident epoch (graph replay friendly); may be null
    unsigned long long* done_flag;                 // host-mapped: last finished epoch on this node (peers' serve loop)
    unsigned long long* idle_ticks;                // host-mapped: launches that gave up waiting for theta (peers re-arm)
    unsigned long long* trace;                     // optional device-timer ring [4 x u64 per epoch % 256] or null
    unsigned long long* cta_trace;                 // optional per-CTA phase stamps [grid][8] of the LAST launch, or null

    // --- low-latency ("LL") mode for small results: flag-in-data words, no fences, no flag writes ----
    // Every 8-byte word carries 32 bits of payload and the low 32 bits of the epoch as its tag, so a
    // reader that sees the right tag has the data (8-byte accesses are single transactions on NVLink
    // and PCIe).  theta: one word per 32-bit theta word; results: two words per double.
    int ll_mode;                                         // results travel as tagged words (small n_vals)
    int ll_theta;                                        // theta travels as tagged words (n_theta <= a few thousand)
    unsigned long long* ll_theta_local;                  // own theta mailbox      [n_theta]
    unsigned long long* ll_peer_theta[B200FED_MAX_WORLD]; // root: every node's     [n_theta]
    unsigned long long* ll_mc_theta;                     // root: multicast alias or null
    unsigned long long* ll_root_slots;                   // root's slot array      [world][n_vals][2]
    unsigned long long* ll_host_result;                  // host-mapped            [n_vals][2]

    // --- speculative root launches (opt-in): the root's kernel is enqueued BEFORE the client has the next theta --
    // The client writes theta as tagged words into host-mapped memory; CTA 0 of the (already resident, set up,
    // first tiles loaded) kernel polls them over PCIe and broadcasts.  If they do not arrive within
    // spec_timeout_ns the launch counts as idle (epoch unchanged, idle tick) exactly like a peer's.
    const unsigned long long* spec_theta;                // host-mapped tagged theta words [n_theta], or null
    unsigned long long* spec_abort;                      // device word: epoch whose speculative launch gave up
    unsigned long long spec_timeout_ns;
};

namespace fed {

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ld_cg_f32(const float* p) {
    float v;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_cg_f64(const double* p) {
    double v;
    asm volatile("ld.global.cg.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// NVSwitch multicast store: one store instruction lands in every node's copy.
__device__ __forceinline__ void multimem_st_f32(float* mc, float v) {
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc), "f"(v) : "memory");
}
__device__ __forceinline__ void multimem_st_release_u64(unsigned long long* mc, unsigned long long v) {
    asm volatile("multimem.st.release.sys.global.u64 [%0], %1;" ::"l"(mc), "l"(v) : "memory");
}

__device__ __forceinline__ void multimem_st_relaxed_u64(unsigned long long* mc, unsigned long long v) {
    asm volatile("multimem.st.relaxed.sys.global.u64 [%0], %1;" ::"l"(mc), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ll_pack(unsigned int payload, unsigned long long epoch) {
    return (unsigned long long)payload | ((epoch & 0xFFFFFFFFull) << 32);
}
// Stores a double as two tagged words.
__device__ __forceinline__ void ll_store_f64(unsigned long long* dst, double v, unsigned long long epoch) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    st_relaxed_sys(dst, ll_pack((unsigned int)bits, epoch));
    st_relaxed_sys(dst + 1, ll_pack((unsigned int)(bits >> 32), epoch));
}
// Polls one tagged word.  0 = ok, 1 = timeout, 2 = STOP seen on the (legacy) flag.
// `abort_flag` (optional): a device word that holds `epoch` once CTA 0 of a speculative launch has given up.
__device__ __forceinline__ int ll_wait_word(const unsigned long long* src, unsigned long long epoch, unsigned long long timeout_ns,
                                            const unsigned long long* stop_flag, unsigned int* payload,
                                            const unsigned long long* abort_flag = nullptr) {
    const unsigned long long want = epoch & 0xFFFFFFFFull;
    unsigned long long t0 = 0;
    unsigned int spins = 0;
    while (true) {
        const unsigned long long w = ld_relaxed_sys(src);
        if ((w >> 32) == want) {
            *payload = (unsigned int)w;
            return 0;
        }
        if ((++spins & 0x3F) == 0) {
            if (t0 == 0) t0 = globaltimer();
            if (stop_flag && (ld_acquire_sys(stop_flag) & B200FED_EPOCH_MASK) == B200FED_STOP_EPOCH) return 2;
            if (abort_flag && ld_acquire_sys(abort_flag) == epoch) return 1;
            if (timeout_ns && globaltimer() - t0 > timeout_ns) return 1;
            __nanosleep(32);
        }
    }
}

// Spin until *flag (epoch part) >= epoch.  Returns false on timeout.
__device__ __forceinline__ bool wait_epoch(const unsigned long long* flag, unsigned long long epoch,
                                           unsigned long long timeout_ns, unsigned long long* seen) {
    unsigned long long t0 = globaltimer();
    unsigned int spins = 0;
    while (true) {
        unsigned long long v = ld_acquire_sys(flag);
        if ((v & B200FED_EPOCH_MASK) >= epoch) {
            *seen = v;
            return true;
        }
        if ((++spins & 0x3F) == 0) {
            if (timeout_ns && globaltimer() - t0 > timeout_ns) {
                *seen = v;
                return false;
            }
            __nanosleep(64);
        }
    }
}

// Per-CTA phase stamp k (0 entry, 1 theta acquired, 2 setup done, 3 first tile landed, 4 last load issued,
// 5 main loop done, 6 partial stored, 7 exit).  Call from ONE thread; a no-op unless tracing is enabled.
__device__ __forceinline__ void stamp(const FedComm& c, int k) {
    if (c.cta_trace) c.cta_trace[(size_t)blockIdx.x * 8 + k] = globaltimer();
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Lets the next kernel of the stream start occupying SMs that this grid no longer needs.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

struct Prologue {
    unsigned long long epoch;   // resolved epoch of this launch
    bool stop;                  // root asked the nodes to drain
    bool timed_out;
};

// Broadcast (root) + acquire (everyone).  Leaves theta[0..n_theta) in `theta_smem`.
// Must be called by all threads of the CTA.
__device__ __forceinline__ Prologue prologue(const FedComm& c, float* theta_smem) {
    __shared__ unsigned long long s_seen;
    __shared__ int s_ok;
    // Programmatic dependent launch: a kernel launched with programmatic stream serialization may become
    // resident while the previous evaluation is still draining (its CTAs called pdl_trigger()); everything
    // above this line (launch, smem carve-up, parameter loads) overlaps with that tail.  The wait returns
    // once the previous grid has completed and its memory operations are visible (no-op otherwise).
    pdl_wait();
    unsigned long long epoch = c.epoch;
    if (c.epoch_counter) epoch = *reinterpret_cast<volatile unsigned long long*>(c.epoch_counter) + 1ull;
    if (threadIdx.x == 0) stamp(c, 0);

    if (c.world == 1 && gridDim.x == 1) {
        // Single node, single CTA (tiny models): no mailbox round trip, no flags — theta goes
        // straight from (host-mapped) memory into shared memory.  Latency path.
        int bad = 0;
        if (c.spec_theta) {
            // speculative launch: theta arrives as tagged words in host memory (or not at all: idle)
            for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) {
                unsigned int payload = 0;
                bad |= ll_wait_word(c.spec_theta + i, epoch, c.spec_timeout_ns, c.flag_local, &payload);
                theta_smem[i] = __uint_as_float(payload);
            }
        } else {
            for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) theta_smem[i] = c.theta_src[i];
        }
        if (threadIdx.x == 0 && c.trace) c.trace[(epoch & 255) * 4 + 0] = globaltimer();
        bad = __syncthreads_or(bad);
        Prologue r0;
        r0.epoch = epoch;
        r0.stop = (bad & 2) != 0;
        r0.timed_out = (bad & 1) != 0;
        return r0;
    }
    if (c.ll_theta) {
        // LL broadcast: tagged theta words, no fence, no flag.  Every thread polls the words it needs.
        if (c.rank == 0 && blockIdx.x == 0) {
            auto fan_out = [&](int i, unsigned long long w) {
                if (c.ll_mc_theta) {
                    multimem_st_relaxed_u64(c.ll_mc_theta + i, w);
                } else {
                    for (int p = 0; p < c.world; ++p) st_relaxed_sys(c.ll_peer_theta[p] + i, w);
                }
            };
            if (c.spec_theta) {
                // speculative launch: every thread polls its own host words (one PCIe round trip once they are
                // written); all or nothing — if any word is missing at the deadline nothing is broadcast and the
                // other CTAs of this GPU are released through the abort word (the peers simply keep waiting)
                constexpr int kSpecPerThread = 8;   // host side: n_theta <= 1024, blocks have >= 128 threads
                unsigned int pay[kSpecPerThread];
                int bad = 0;
#pragma unroll
                for (int k = 0; k < kSpecPerThread; ++k) {
                    const int i = threadIdx.x + k * blockDim.x;
                    pay[k] = 0;
                    if (i < c.n_theta) bad |= ll_wait_word(c.spec_theta + i, epoch, c.spec_timeout_ns, c.flag_local, &pay[k]);
                }
                bad = __syncthreads_or(bad);
                if (!bad) {
#pragma unroll
                    for (int k = 0; k < kSpecPerThread; ++k) {
                        const int i = threadIdx.x + k * blockDim.x;
                        if (i < c.n_theta) fan_out(i, ll_pack(pay[k], epoch));
                    }
                } else if (threadIdx.x == 0 && !(bad & 2)) {
                    st_release_sys(c.spec_abort, epoch);
                }
            } else {
                for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) fan_out(i, ll_pack(__float_as_uint(c.theta_src[i]), epoch));
            }
            if (threadIdx.x == 0 && c.trace) c.trace[(epoch & 255) * 4 + 0] = globaltimer();
        }
        if (threadIdx.x == 0) s_ok = 0;
        __syncthreads();
        int bad = 0;
        for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) {
            unsigned int payload = 0;
            const int rc = ll_wait_word(c.ll_theta_local + i, epoch, c.timeout_ns, c.flag_local, &payload,
                                        c.spec_theta ? c.spec_abort : nullptr);
            if (rc) bad |= rc;
            theta_smem[i] = __uint_as_float(payload);
        }
        if (bad) atomicOr(&s_ok, bad);
        __syncthreads();
        Prologue rl;
        rl.epoch = epoch;
        rl.timed_out = (s_ok & 1) != 0;
        rl.stop = (s_ok & 2) != 0;
        __syncthreads();
        if (threadIdx.x == 0) stamp(c, 1);
        return rl;
    }
    if (c.rank == 0 && blockIdx.x == 0) {
        // theta_src may live in host memory: read it once, fan it out over NVLink.
        for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) {
            float v = c.theta_src[i];
            if (c.mc_theta) {
                multimem_st_f32(c.mc_theta + i, v);
            } else {
                for (int p = 0; p < c.world; ++p) c.peer_theta[p][i] = v;
            }
        }
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0 && c.trace) c.trace[(epoch & 255) * 4 + 0] = globaltimer();
        if (c.mc_flag) {
            if (threadIdx.x == 0) multimem_st_release_u64(c.mc_flag, epoch);
        } else if (threadIdx.x < c.world) {
            // one releasing thread per node: the system-scope fences run in parallel, not in series
            st_release_sys(c.peer_flag[threadIdx.x], epoch);
        }
    }
    if (threadIdx.x == 0) {
        unsigned long long seen = 0;
        s_ok = wait_epoch(c.flag_local, epoch, c.timeout_ns, &seen) ? 1 : 0;
        s_seen = seen;
    }
    __syncthreads();
    Prologue r;
    r.epoch = epoch;
    r.timed_out = (s_ok == 0);
    r.stop = ((s_seen & B200FED_EPOCH_MASK) == B200FED_STOP_EPOCH);
    if (!r.timed_out && !r.stop) {
        for (int i = threadIdx.x; i < c.n_theta; i += blockDim.x) theta_smem[i] = ld_cg_f32(c.theta_local + i);
    }
    __syncthreads();
    if (threadIdx.x == 0) stamp(c, 1);
    return r;
}

// ---- double-double partial sums --------------------------------------------------------------------------
// Kernels that hand out work dynamically (csrc/glm_tc.cu) cannot fix WHICH CTA sums which chunk of rows, so
// they keep every running sum as an unevaluated pair (hi, lo) with |lo| <= ulp(hi)/2 (Knuth TwoSum).  Every
// chunk contributes a value that depends on the chunk only; pairs make the additions exact to ~2^-100, so the
// total — rounded to a double exactly once, at the very end — does not depend on the assignment of chunks to
// CTAs (bit-reproducible except when the exact sum sits within 2^-100 of a rounding boundary).
__device__ __forceinline__ void dd_add(double& hi, double& lo, double xh, double xl) {
    const double s = hi + xh;
    const double bb = s - hi;
    const double err = (hi - (s - bb)) + (xh - bb);
    hi = s;
    lo += err + xl;
}
__device__ __forceinline__ double2 ld_cg_f64x2(const double* p) {
    double2 v;
    asm volatile("ld.global.cg.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p) : "memory");
    return v;
}

constexpr unsigned int kReduceGroup = 16;   // CTAs per level-1 reduction group

// Fixed-order sum of value v over rows [first, first + count) of a partial array with `stride` doubles per
// row.  DD: rows hold (hi, lo) pairs and the result is a pair; otherwise plain doubles (lo stays 0).  kWideDD: (hi, lo)
// pairs of loads in flight per thread; the order of the additions does not depend on it.
template <bool DD, unsigned int kWideDD = 16>
__device__ __forceinline__ void sum_rows(const double* rows, size_t stride, int v, unsigned int first, unsigned int count,
                                         double& hi, double& lo) {
    constexpr unsigned int kWide = DD ? kWideDD : 37;   // loads in flight per thread
    hi = 0.0;
    lo = 0.0;
    for (unsigned int b = 0; b < count; b += kWide) {
        if constexpr (DD) {
            double2 t[kWide];
#pragma unroll
            for (unsigned int j = 0; j < kWide; ++j)
                t[j] = (b + j < count) ? ld_cg_f64x2(rows + (size_t)(first + b + j) * stride + 2 * (size_t)v) : make_double2(0.0, 0.0);
#pragma unroll
            for (unsigned int j = 0; j < kWide; ++j) dd_add(hi, lo, t[j].x, t[j].y);
        } else {
            double t[kWide];
#pragma unroll
            for (unsigned int j = 0; j < kWide; ++j)
                t[j] = (b + j < count) ? ld_cg_f64(rows + (size_t)(first + b + j) * stride + v) : 0.0;
#pragma unroll
            for (unsigned int j = 0; j < kWide; ++j) hi += t[j];
        }
    }
}

// Every CTA has stored its partial into row blockIdx.x of c.cta_partials (`row_stride` doubles per row; DD:
// (hi, lo) pairs).  Two-level, fixed-shape reduction: the last CTA to finish within a group of kReduceGroup
// consecutive CTAs sums the group's rows into `group_buf[group]` (groups that finish early reduce early, off
// the critical path); the last group to finish sums the group partials, exchanges the node partial with the
// root over NVLink, and the root publishes the result to the host.  Returns true in the one CTA that ran the
// final stage (it may reset per-launch kernel state such as work counters).  Must be called by all threads.
// kWideDD: see sum_rows (a kernel that runs at 128 registers per thread needs fewer than 16 pairs in flight).
template <bool DD, unsigned int kWideDD = 16>
__device__ __forceinline__ bool epilogue_t(const FedComm& c, const Prologue& pro, unsigned long long status_in,
                                           size_t row_stride, double* group_buf) {
    __shared__ int s_last;
    __shared__ unsigned long long s_status;
    const int nv = c.n_vals;
    if (c.world == 1 && gridDim.x == 1) {
        // latency path: the only CTA's partial IS the result
        __syncthreads();
        if (pro.timed_out || pro.stop) {
            // a speculative launch whose theta never came: idle (epoch unchanged, the host counts the tick)
            if (threadIdx.x == 0) {
                if (pro.timed_out && !pro.stop && c.spec_theta && c.idle_ticks) {
                    volatile unsigned long long* ticks = c.idle_ticks;
                    *ticks = *ticks + 1ull;
                } else if (c.host_flag) {
                    __threadfence_system();
                    st_release_sys(c.host_flag, (pro.stop ? B200FED_STOP_EPOCH : pro.epoch) |
                                                    ((pro.stop ? 0ull : B200FED_ERR_THETA_TIMEOUT) << B200FED_STATUS_SHIFT));
                }
            }
            return true;
        }
        auto value = [&](int v) { return DD ? c.cta_partials[2 * v] + c.cta_partials[2 * v + 1] : c.cta_partials[v]; };
        if (c.ll_mode) {
            // tagged words straight to host-mapped memory: no fence, no flag
            for (int v = threadIdx.x; v < nv; v += blockDim.x) ll_store_f64(c.ll_host_result + 2 * v, value(v), pro.epoch);
            if (threadIdx.x == 0) {
                if (c.trace) {
                    c.trace[(pro.epoch & 255) * 4 + 1] = globaltimer();
                    c.trace[(pro.epoch & 255) * 4 + 2] = globaltimer();
                }
                if (c.epoch_counter) *c.epoch_counter = pro.epoch;
                if (c.done_flag) *reinterpret_cast<volatile unsigned long long*>(c.done_flag) = pro.epoch;
                stamp(c, 7);
            }
            return true;
        }
        for (int v = threadIdx.x; v < nv; v += blockDim.x) c.host_result[v] = value(v);
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (c.trace) {
                c.trace[(pro.epoch & 255) * 4 + 1] = globaltimer();
                c.trace[(pro.epoch & 255) * 4 + 2] = globaltimer();
            }
            st_release_sys(c.host_flag, pro.epoch | (status_in << B200FED_STATUS_SHIFT));
            if (c.epoch_counter) *c.epoch_counter = pro.epoch;
            if (c.done_flag) *reinterpret_cast<volatile unsigned long long*>(c.done_flag) = pro.epoch;
            stamp(c, 7);
        }
        return true;
    }
    const bool computed = !(pro.stop || pro.timed_out);
    const unsigned int n_groups = (gridDim.x + kReduceGroup - 1) / kReduceGroup;
    const unsigned int grp = blockIdx.x / kReduceGroup;
    const unsigned int grp_first = grp * kReduceGroup;
    const unsigned int grp_size = min(kReduceGroup, gridDim.x - grp_first);
    constexpr int kW = DD ? 2 : 1;

    // ---- level 1: last CTA of the group -> group partial ------------------------------------------------
    // any CTA's fault reaches the final stage — and so does any CTA's expired wait for theta: the bounded waits
    // run out per CTA, so when theta arrives right at the deadline some CTAs may have computed and others not
    const unsigned long long status_cta = status_in | ((pro.timed_out && !pro.stop) ? B200FED_ERR_THETA_TIMEOUT : 0ull);
    if (threadIdx.x == 0 && status_cta) atomicOr(c.ticket + 255, (unsigned int)status_cta);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(c.ticket + 1 + grp, 1u);
        s_last = (t == grp_size - 1) ? 1 : 0;
        if (s_last) c.ticket[1 + grp] = 0;   // nobody touches this group's ticket again in this launch
        s_status = status_in;
    }
    __syncthreads();
    if (!s_last) {
        if (threadIdx.x == 0) stamp(c, 7);
        return false;
    }
    __threadfence();
    if (computed) {
        for (int v = threadIdx.x; v < nv; v += blockDim.x) {
            double hi, lo;
            sum_rows<DD, kWideDD>(c.cta_partials, row_stride, v, grp_first, grp_size, hi, lo);
            group_buf[((size_t)grp * nv + v) * kW] = hi;
            if constexpr (DD) group_buf[((size_t)grp * nv + v) * kW + 1] = lo;
        }
    }
    // ---- level 2: last group -> node partial ------------------------------------------------------------
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(c.ticket, 1u);
        s_last = (t == n_groups - 1) ? 1 : 0;
    }
    __syncthreads();
    if (!s_last) {
        if (threadIdx.x == 0) stamp(c, 7);
        return false;
    }
    __threadfence();
    const unsigned long long epoch = pro.epoch;
    if (threadIdx.x == 0) {
        s_status |= (unsigned long long)atomicExch(c.ticket + 255, 0u);
    }
    __syncthreads();
    // The evaluation counts only if EVERY CTA had theta.  A mixed launch (see above) is treated like an expired
    // wait: nothing is published; a peer leaves the epoch where it was, the serve loop re-arms it, and the next
    // kernel finds this epoch's theta already in its mailbox and recomputes.
    const bool any_timed_out = (s_status & B200FED_ERR_THETA_TIMEOUT) != 0ull;

    if (!computed || any_timed_out) {
        // nothing was computed: just report and drain.  A PEER whose wait for theta expired has merely been idle
        // (the client paused between evaluations): it leaves the epoch where it was and counts an idle tick, so
        // the serve loop re-arms it instead of taking the federation down.
        if (threadIdx.x == 0) {
            const bool timed_out = pro.timed_out || any_timed_out;
            // (the root of a speculative launch is in the same position as a peer: the client was not ready)
            const bool idle = timed_out && !pro.stop && (c.rank != 0 || c.spec_theta != nullptr);
            if (idle && c.rank == 0) *c.spec_abort = 0ull;   // the next launch of this epoch starts clean
            const unsigned long long done_epoch = idle ? epoch - 1ull : epoch;
            *c.ticket = 0;
            if (c.epoch_counter) *c.epoch_counter = done_epoch;
            unsigned long long st = (timed_out && !idle) ? B200FED_ERR_THETA_TIMEOUT : 0ull;
            unsigned long long word = (pro.stop ? B200FED_STOP_EPOCH : done_epoch) | (st << B200FED_STATUS_SHIFT);
            if (idle && c.idle_ticks) {
                volatile unsigned long long* ticks = c.idle_ticks;
                *ticks = *ticks + 1ull;
            }
            if (c.done_flag) { *reinterpret_cast<volatile unsigned long long*>(c.done_flag) = word; }
            if (c.rank == 0 && c.host_flag) {
                __threadfence_system();
                st_release_sys(c.host_flag, word);
            }
        }
        return true;
    }
    auto node_value = [&](int v) {
        double hi, lo;
        sum_rows<DD, kWideDD>(group_buf, (size_t)nv * kW, v, 0u, n_groups, hi, lo);
        return hi + lo;   // DD: the one rounding of this node's partial
    };

    if (c.ll_mode) {
        // LL reduce: each node's last CTA stores tagged words into the root's slot array (NVLink, no fence,
        // no flag); the root polls the words of every node in rank order, sums, and stores tagged words into
        // host-mapped memory.
        unsigned long long* my_slot_ll = c.ll_root_slots + (size_t)c.rank * nv * 2;
        for (int v = threadIdx.x; v < nv; v += blockDim.x) {
            const double s = node_value(v);
            if (c.rank != 0) {
                ll_store_f64(my_slot_ll + 2 * v, s, epoch);
            } else {
                double total = s;  // rank 0 first, then the peers in rank order
                bool ok = true;
                for (int p = 1; p < c.world && ok; ++p) {
                    unsigned int lo = 0, hi = 0;
                    const unsigned long long* src = c.ll_root_slots + ((size_t)p * nv + v) * 2;
                    ok = ll_wait_word(src, epoch, c.timeout_ns, nullptr, &lo) == 0 &&
                         ll_wait_word(src + 1, epoch, c.timeout_ns, nullptr, &hi) == 0;
                    total += __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
                }
                if (ok) ll_store_f64(c.ll_host_result + 2 * v, total, epoch);
                else atomicOr(&s_status, B200FED_ERR_PEER_TIMEOUT);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (c.trace) {
                c.trace[(epoch & 255) * 4 + 1] = globaltimer();
                if (c.rank == 0) c.trace[(epoch & 255) * 4 + 2] = globaltimer();
            }
            if (c.rank == 0 && s_status) {  // errors travel on the legacy flag (the tagged words stay incomplete)
                __threadfence_system();
                st_release_sys(c.host_flag, epoch | (s_status << B200FED_STATUS_SHIFT));
            }
            *c.ticket = 0;
            if (c.epoch_counter) *c.epoch_counter = epoch;
            if (c.done_flag) *reinterpret_cast<volatile unsigned long long*>(c.done_flag) = epoch | (s_status << B200FED_STATUS_SHIFT);
            stamp(c, 7);
        }
        return true;
    }

    if (c.rank != 0) {
        // peer: node partial -> root's slot for this rank (NVLink stores), then the slot flag
        double* my_slot = c.root_slots + (size_t)c.rank * nv;
        for (int v = threadIdx.x; v < nv; v += blockDim.x) my_slot[v] = node_value(v);
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (c.trace) c.trace[(epoch & 255) * 4 + 1] = globaltimer();
            st_release_sys(c.root_slot_flags + c.rank, epoch);
        }
    } else {
        // root: own partial stays in registers; gather the peers, ordered sum (rank 0, 1, 2, ...), publish
        if (threadIdx.x == 0 && c.trace) c.trace[(epoch & 255) * 4 + 1] = globaltimer();
        constexpr int kOwn = 4;   // values per thread kept in registers across the wait for the peers
        double own[kOwn];
        const bool cached = nv <= kOwn * (int)blockDim.x;
        if (cached) {
#pragma unroll
            for (int i = 0; i < kOwn; ++i) {
                const int v = threadIdx.x + i * blockDim.x;
                own[i] = v < nv ? node_value(v) : 0.0;
            }
        }
        if (threadIdx.x >= 1 && threadIdx.x < c.world) {
            unsigned long long seen;
            bool ok = wait_epoch(c.root_slot_flags + threadIdx.x, epoch, c.timeout_ns, &seen);
            if (!ok) atomicOr(&s_status, B200FED_ERR_PEER_TIMEOUT);
        }
        __syncthreads();
        if (cached) {
#pragma unroll
            for (int i = 0; i < kOwn; ++i) {
                const int v = threadIdx.x + i * blockDim.x;
                if (v < nv) {
                    double s = own[i];
                    for (int p = 1; p < c.world; ++p) s += ld_cg_f64(c.root_slots + (size_t)p * nv + v);
                    c.host_result[v] = s;
                }
            }
        } else {
            for (int v = threadIdx.x; v < nv; v += blockDim.x) {
                double s = node_value(v);
                for (int p = 1; p < c.world; ++p) s += ld_cg_f64(c.root_slots + (size_t)p * nv + v);
                c.host_result[v] = s;
            }
        }
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (c.trace) c.trace[(epoch & 255) * 4 + 2] = globaltimer();
            st_release_sys(c.host_flag, epoch | (s_status << B200FED_STATUS_SHIFT));
        }
    }
    if (threadIdx.x == 0) {
        *c.ticket = 0;
        if (c.epoch_counter) *c.epoch_counter = epoch;
        if (c.done_flag) *reinterpret_cast<volatile unsigned long long*>(c.done_flag) = epoch | (s_status << B200FED_STATUS_SHIFT);
        stamp(c, 7);
    }
    return true;
}

// Plain-double partials, one row of n_vals per CTA (every kernel except the dynamically scheduled GLM).
__device__ __forceinline__ bool epilogue(const FedComm& c, const Prologue& pro, unsigned long long status_in) {
    return epilogue_t<false>(c, pro, status_in, (size_t)c.n_vals, c.group_partials);
}

// Order-independent accumulation for values that many threads add to one shared cell (the
// per-group intercept gradients): 40.24 fixed point in a 64-bit integer.  Integer addition is
// associative, so the result does not depend on which thread's atomic lands first — unlike
// floating-point atomics — and evaluations stay bit-reproducible.  Resolution 6e-8, range +-5e11.
__device__ __forceinline__ void fix_add(unsigned long long* acc, double v) {
    atomicAdd(acc, (unsigned long long)__double2ll_rn(v * 16777216.0));
}
__device__ __forceinline__ double fix_get(unsigned long long a) { return (double)(long long)a * (1.0 / 16777216.0); }

// block-wide sum of doubles; result valid in thread 0.  `buf` needs >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* buf) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) buf[w] = v;
    __syncthreads();
    if (w == 0) {
        v = (l < (int)((blockDim.x + 31) >> 5)) ? buf[l] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    return v;
}

}  // namespace fed
