// sph_dfsph.cuh -- divergence-free SPH (reference DFSPH.py, simulationMethod 4) on top of the same
// sorted SoA state and per-step neighbour lists as the WCSPH path.
//
// compute_densities (DFSPH.py:39-47) is k_density_tma in DFSPH mode (no clamp, no EOS); it also
// builds the neighbour lists that every kernel below walks.  Each kernel here is one reference @ti.kernel.
// The convergence loops (divergence_solve / pressure_solve, DFSPH.py:236-276, 314-352) exist twice: in the Python
// shell exactly as the reference writes them (one density-error read-back per Jacobi sweep), and as
// sph_dfsph_solve: the sweeps of a batch are launched back to back, the loop condition is evaluated ON THE
// DEVICE by k_dfsph_check after every sweep (DfsphCtrl), and the sweeps behind the converged one return at once --
// same sweeps, same iteration counts, one read-back per batch instead of one per sweep.
#pragma once
#include "sph_kernels.cuh"

enum DfsphOp {
    DFSPH_COMPUTE_DENSITIES = 0,   // DFSPH.py:39-47
    DFSPH_COMPUTE_FACTOR = 1,      // DFSPH.py:114-139
    DFSPH_DENSITY_CHANGE = 2,      // DFSPH.py:157-178
    DFSPH_DENSITY_ADV = 3,         // DFSPH.py:198-205
    DFSPH_DENSITY_ERROR = 4,       // DFSPH.py:221-227   (arg = offset, out = double accumulator)
    DFSPH_MULTIPLY_FACTOR = 5,     // DFSPH.py:229-233 on dfsph_factor (arg = time_step)
    DFSPH_DIVERGENCE_ITERATION = 6,// DFSPH.py:278-290
    DFSPH_PRESSURE_ITERATION = 7,  // DFSPH.py:354-367
    DFSPH_NON_PRESSURE_FORCES = 8, // DFSPH.py:92-101
    DFSPH_PREDICT_VELOCITY = 9,    // DFSPH.py:392-397
    DFSPH_ADVECT = 10,             // DFSPH.py:104-111
};

// Device-resident state of one convergence loop (sph_dfsph_solve); lives in the workspace scratch block.
struct DfsphCtrl {
    double err;          // running sum of (rho0 * density_adv - offset) of the current sweep
    double last_avg;     // avg_density_err of the last evaluated sweep
    int32_t iterations;  // the reference's m_iterations(_v): sweeps that did NOT meet eta
    int32_t done;        // loop left (converged, or the iteration cap reached)
    int32_t sweeps;      // sweeps actually executed
    int32_t err_max;     // PCISPH: the running max of the sweep's error, as the int bits of a non-negative float
};

// Dense walk over the neighbour list of particle i (reference visiting order), gathers batched by
// four; falls back to the 27-cell scan when the list overflowed.  fn(j, rx, ry, rz, r2, posm_j).
template <typename F>
__device__ __forceinline__ void for_listed_neighbors(const DevParams &P, const DevArrays &S, int i, const float4 &pi,
                                                     F &&fn) {
    const int cnt = S.nbr_cnt[i];
    if (cnt != NBR_OVERFLOW) {
        const int32_t *lp = S.nbr_list + i;
        const size_t stride = (size_t)S.npad;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            int j[4];
            float4 pj[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                j[u] = (k0 + u < cnt) ? lp[(size_t)(k0 + u) * stride] : i;
                pj[u] = __ldg(S.posm + j[u]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (k0 + u < cnt) {
                    float rx = pi.x - pj[u].x, ry = pi.y - pj[u].y, rz = pi.z - pj[u].z;
                    fn(j[u], rx, ry, rz, rx * rx + ry * ry + rz * rz, pj[u]);
                }
            }
        }
    } else {
        for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z, fn);
    }
}

// x-slab sharding: P.n is the capacity, and every per-particle DFSPH kernel but the density pass works on the
// owned index range of the device step state only (ghosts are neighbours; their values come from the owner)
__device__ __forceinline__ bool dfsph_in_range(const DevParams &P, const DevArrays &S, int i) {
    if (i >= P.n) return false;
    return !P.slab_on || (i >= S.sd[SD_OWN0] && i < S.sd[SD_OWN1]);
}

__device__ __forceinline__ bool dfsph_fluid(const DevParams &P, const DevArrays &S, int i, uint32_t &fl) {
    if (!dfsph_in_range(P, S, i)) return false;
    fl = __float_as_uint(S.misc[i].z);
    return (fl & FLAG_FLUID) != 0;
}

// grad W(x_i - x_j) = gs * r
__device__ __forceinline__ float gradw_of(const DevParams &P, float r2) {
    float r, inv_r;
    fast_norm(r2, r, inv_r);
    return gradw_scale_fast(P, r, inv_r);
}

// DFSPH.py:114-154
__global__ void __launch_bounds__(128) k_dfsph_factor(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    float4 pi = S.posm[i];
    float gx = 0.f, gy = 0.f, gz = 0.f, sum_k = 0.f;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        float s = -pj.w * gradw_of(P, r2);  // grad_p_j = -m_V_j * grad W
        float ax = s * rx, ay = s * ry, az = s * rz;
        if (__ldg(&S.aux[j].z) > 0.0f) sum_k += ax * ax + ay * ay + az * az;  // fluid neighbours only
        gx -= ax; gy -= ay; gz -= az;
    });
    sum_k += gx * gx + gy * gy + gz * gz;
    S.dfs[i].x = (sum_k > 1e-6f) ? -1.0f / sum_k : 0.0f;
}

// MODE 0: compute_density_change (DFSPH.py:157-196);  MODE 1: compute_density_adv (DFSPH.py:198-219)
template <int MODE>
__device__ __forceinline__ float dfsph_density_change_of(const DevParams &P, const DevArrays &S, int i) {
    float4 pi = S.posm[i];
    float4 vi = S.veld[i];
    float acc = 0.f;
    int nn = 0;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        float4 vj = __ldg(S.veld + j);
        float gs = gradw_of(P, r2);
        acc += pj.w * (((vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz) * gs);
        ++nn;
    });
    float da;
    if (MODE == 0) {
        da = fmaxf(acc, 0.0f);        // only correct positive divergence
        if (nn < 20) da = 0.0f;       // particle deficiency (3-D)
    } else {
        da = fmaxf(vi.w / P.rho0 + P.dt * acc, 1.0f);
    }
    S.dfs[i].y = da;
    return da;
}
template <int MODE>
__global__ void __launch_bounds__(128) k_dfsph_density_change(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    dfsph_density_change_of<MODE>(P, S, i);
}

// block-wide fp64 sum -> one atomic per CTA (DFSPH.py:221-227 returns the sum to the host)
template <int WARPS>
__device__ __forceinline__ void dfsph_block_sum_to(double e, double *out) {
    __shared__ double red[WARPS];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = threadIdx.x < WARPS ? red[threadIdx.x] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) atomicAdd(out, t);
    }
}

// One sweep of sph_dfsph_solve = k_dfsph_iteration + this kernel + k_dfsph_check: the density change / advected
// density of the sweep and its error sum in ONE pass (the host loop runs compute_density_error as a second kernel).
template <int MODE>
__global__ void __launch_bounds__(128) k_dfsph_density_change_err(DevParams P, DevArrays S, float offset, DfsphCtrl *ctrl) {
    if (ctrl->done) return;  // written only by k_dfsph_check, between kernels: uniform over the grid
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    double e = 0.0;
    if (dfsph_fluid(P, S, i, fl)) e = (double)(P.rho0 * dfsph_density_change_of<MODE>(P, S, i) - offset);
    dfsph_block_sum_to<4>(e, &ctrl->err);
}

// The loop condition of divergence_solve / pressure_solve (DFSPH.py:245-254, 323-331), evaluated on the device:
//   while m < 1 or m < max_iterations:  avg = sweep();  if avg <= eta: break;  m += 1
__device__ __forceinline__ void dfsph_check_sum(DfsphCtrl *ctrl, double err, double n_fluid, double eta,
                                                int32_t max_iterations) {
    const double avg = err / n_fluid;
    ctrl->last_avg = avg;
    ctrl->err = 0.0;
    ctrl->sweeps += 1;
    if (avg <= eta) { ctrl->done = 1; return; }
    const int32_t m = ctrl->iterations + 1;
    ctrl->iterations = m;
    if (!(m < 1 || m < max_iterations)) ctrl->done = 1;
}
__global__ void k_dfsph_check(DfsphCtrl *ctrl, double n_fluid, double eta, int32_t max_iterations) {
    if (ctrl->done) return;
    dfsph_check_sum(ctrl, ctrl->err, n_fluid, eta, max_iterations);
}
// Sharded loops: parts[r] holds rank r's error partial (this rank's own is still in ctrl->err), all-gathered over the
// transport.  The partials are summed in RANK order, so every rank computes a bit-identical sum -- and from it the
// same avg / done / iterations -- and issues the same number of transport calls.
__device__ __forceinline__ double ranked_err_sum(const DfsphCtrl *ctrl, const double *parts, int32_t rank, int32_t world) {
    double err = rank == 0 ? ctrl->err : parts[0];
    for (int r = 1; r < world; ++r) err += r == rank ? ctrl->err : parts[r];
    return err;
}
__global__ void k_dfsph_check_ranked(DfsphCtrl *ctrl, const double *parts, int32_t rank, int32_t world, double n_fluid,
                                     double eta, int32_t max_iterations) {
    if (ctrl->done) return;
    dfsph_check_sum(ctrl, ranked_err_sum(ctrl, parts, rank, world), n_fluid, eta, max_iterations);
}

// DFSPH.py:221-227
__global__ void __launch_bounds__(256) k_dfsph_density_error(DevParams P, DevArrays S, float offset, double *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    uint32_t fl;
    if (dfsph_fluid(P, S, i, fl)) e = (double)(P.rho0 * S.dfs[i].y - offset);
    dfsph_block_sum_to<8>(e, out);
}

// DFSPH.py:229-233 applied to dfsph_factor
__global__ void k_dfsph_multiply_factor(DevParams P, DevArrays S, float ts) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    S.dfs[i].x *= ts;
}

// MODE 0: divergence_solver_iteration_kernel (DFSPH.py:278-311);  MODE 1: pressure_solve_iteration_kernel
// (DFSPH.py:354-389).  The reactions MODE 0 would add to dynamic rigid particles are overwritten by
// compute_non_pressure_forces before anything reads them (DFSPH.py:402), so only MODE 1 scatters them.
template <int MODE>
__global__ void __launch_bounds__(128) k_dfsph_iteration(DevParams P, DevArrays S, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;  // sph_dfsph_solve: a sweep launched behind the converged one
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    const float eps = 1e-5f;
    const float boff = MODE == 0 ? 0.0f : 1.0f;
    float4 pi = S.posm[i];
    float4 vi = S.veld[i];
    float4 di = S.dfs[i];
    const float k_i = (di.y - boff) * di.x;
    float dvx = 0.f, dvy = 0.f, dvz = 0.f;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        float4 aj = __ldg(S.aux + j);
        if (aj.z > 0.0f) {  // fluid neighbour
            float4 dj = __ldg(S.dfs + j);
            float k_sum = k_i + (dj.y - boff) * dj.x;
            if (fabsf(k_sum) > eps) {
                float s = -pj.w * gradw_of(P, r2);  // grad_p_j = s * r
                float c = P.dt * k_sum * s;
                if (MODE == 0) { dvx -= c * rx; dvy -= c * ry; dvz -= c * rz; }
                else { vi.x -= c * rx; vi.y -= c * ry; vi.z -= c * rz; }
            }
        } else if (fabsf(k_i) > eps) {  // boundary neighbour (Akinci 2012)
            float s = -pj.w * gradw_of(P, r2);
            float c = -P.dt * 1.0f * k_i * s;  // vel_change = c * r
            if (MODE == 0) { dvx += c * rx; dvy += c * ry; dvz += c * rz; }
            else {
                vi.x += c * rx; vi.y += c * ry; vi.z += c * rz;
                if (aj.z < -1.5f) {  // dynamic rigid body: reaction, DFSPH.py:388-389
                    float f = -(1.0f / P.dt) * vi.w / aj.x;
                    float *a = reinterpret_cast<float *>(S.acc + j);
                    atomicAdd(a + 0, c * rx * f);
                    atomicAdd(a + 1, c * ry * f);
                    atomicAdd(a + 2, c * rz * f);
                }
            }
        }
    });
    if (MODE == 0) { vi.x += dvx; vi.y += dvy; vi.z += dvz; }
    S.veld[i] = vi;
}

// compute_non_pressure_forces (DFSPH.py:50-101): cohesion + viscosity, list based
__global__ void __launch_bounds__(128) k_dfsph_non_pressure(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!dfsph_in_range(P, S, i)) return;
    float4 mi = S.misc[i];
    uint32_t fl = __float_as_uint(mi.z);
    if (!(fl & FLAG_FLUID)) {
        bool dyn = (fl & FLAG_DYNAMIC) != 0;
        S.acc[i] = dyn ? make_float4(P.gx_, P.gy_, P.gz_, 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    float4 pi = S.posm[i];
    float4 vi = S.veld[i];
    const float coh_i = P.sigma / mi.x;
    float ax = P.gx_, ay = P.gy_, az = P.gz_;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        float4 aj = __ldg(S.aux + j);
        if (aj.z > 0.0f) {
            float r, inv_r;
            fast_norm(r2, r, inv_r);
            float w = (r2 > P.d2) ? w_cubic(P, r) : P.w_diam;
            float c = coh_i * aj.z;
            ax -= c * rx * w; ay -= c * ry * w; az -= c * rz * w;
            float4 vj = __ldg(S.veld + j);
            float vxy = (vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz;
            float sv = __fdividef(P.d_visc * aj.x * vxy, r * r + P.visc_eps) * gradw_scale_fast(P, r, inv_r);
            ax += sv * rx; ay += sv * ry; az += sv * rz;
        }
    });
    S.acc[i] = make_float4(ax, ay, az, 0.f);
}

// DFSPH.py:392-397
__global__ void k_dfsph_predict_velocity(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl) || !(fl & FLAG_DYNAMIC)) return;
    float4 v = S.veld[i], a = S.acc[i];
    v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    S.veld[i] = v;
}

// DFSPH.py:104-111.  Sharded: the end-of-step exchange only carries the cell layers next to a cut, so a particle
// that moves a whole cell layer in x within one step could be lost -- flagged instead (SPH_STATUS_SHARD_VELOCITY).
__global__ void k_dfsph_advect(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!dfsph_in_range(P, S, i)) return;
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i];
    if (!(fl & FLAG_FLUID)) {
        float4 a = S.acc[i];
        v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
        S.veld[i] = v;
    }
    if (P.slab_on && !(fabsf(v.x) * P.dt < P.h)) atomicOr(S.status, SPH_STATUS_SHARD_VELOCITY);
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    S.posm[i] = p;
}

// ---- x-slab sharding of the DFSPH step (sph_shard_dfsph_step) ----------------------------------------------------
// Index ranges of the sorted arrays that the per-step ghost alignment and the per-sweep exchanges work on
// (DevArrays::sd holds the WCSPH step state; these live in a separate block of the shard buffer).
enum {
    DX_SEND_L0 = 0, DX_SEND_L1, DX_SEND_L1E,  // to the left: owned layers [sx0, sx0 + sgw), the first ends at L1E
    DX_SEND_R0, DX_SEND_R1, DX_SEND_R1B,      // to the right: owned layers [sx1 - sgw, sx1), the last starts at R1B
    DX_GHOST_L0, DX_GHOST_L1, DX_GHOST_L1B,   // ghost layers [sx0 - sgw, sx0), the first ghost layer starts at L1B
    DX_GHOST_R0, DX_GHOST_R1, DX_GHOST_R1E,   // ghost layers [sx1, sx1 + sgw), the first ghost layer ends at R1E
    DX_HDR_SEND = 16,                         // 4 ints per side: {records of the sgw layers, records of the first}
    DX_HDR_RECV = 32,                         // the same, received from the left / right neighbour
    DX_INTS = 64
};
// what a pack / unpack moves: the alignment, or one 16-byte word per particle of one per-step array (DFSPH: veld, dfs;
// IISPH: veld, acc = {a^p, fluid mark}, aux = {.., p / rho^2, ..}; IISPH with dynamic solids, once after the loop:
// misc, of which only .y = the final pressure p lands on the ghost)
enum { DX_ALIGN = 0, DX_VELD = 1, DX_DFS = 2, DX_ACC = 3, DX_AUX = 4, DX_MISC = 5 };

__device__ __forceinline__ float4 *dx_sweep_array(const DevArrays &S, int what) {
    return what == DX_VELD ? S.veld : what == DX_DFS ? S.dfs : what == DX_ACC ? S.acc : what == DX_MISC ? S.misc : S.aux;
}

// After k_shard_info: the ranges above, and the alignment headers.  A range longer than its message capacity is cut
// and flagged (SPH_STATUS_HALO_CAPACITY), never written out of bounds.
__global__ void k_dfsph_shard_ranges(DevParams P, DevArrays S, int32_t *dx, int align_cap, int sweep_cap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int32_t *sd = S.sd;
    const int layer = P.gy * P.gz;
    const int sx0 = sd[SD_SX0], sx1 = sd[SD_SX1], o0 = sd[SD_OWN0], o1 = sd[SD_OWN1];
    auto start_of_layer = [&](int L) {
        L = min(max(L, 0), P.gx);
        int c = L * layer;
        return c > 0 ? S.cell_end[c - 1] : 0;
    };
    int sl1 = start_of_layer(min(sx0 + P.sgw, sx1)), sl1e = start_of_layer(min(sx0 + 1, sx1));
    int sr0 = start_of_layer(max(sx1 - P.sgw, sx0)), sr1b = start_of_layer(max(sx1 - 1, sx0));
    int gl0 = start_of_layer(sx0 - P.sgw), gl1b = start_of_layer(sx0 - 1);
    int gr1 = start_of_layer(sx1 + P.sgw), gr1e = start_of_layer(sx1 + 1);
    if (!P.has_left) { sl1 = sl1e = o0; gl0 = gl1b = o0; }
    if (!P.has_right) { sr0 = sr1b = o1; gr1 = gr1e = o1; }
    uint32_t flags = 0u;
    if (sl1 - o0 > align_cap) { sl1 = o0 + align_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (o1 - sr0 > align_cap) { sr0 = o1 - align_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (o0 - gl0 > align_cap) { gl0 = o0 - align_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (gr1 - o1 > align_cap) { gr1 = o1 + align_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    sl1e = min(sl1e, sl1); sr1b = max(sr1b, sr0); gl1b = max(gl1b, gl0); gr1e = min(gr1e, gr1);
    if (sl1e - o0 > sweep_cap) { sl1e = o0 + sweep_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (o1 - sr1b > sweep_cap) { sr1b = o1 - sweep_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (o0 - gl1b > sweep_cap) { gl1b = o0 - sweep_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (gr1e - o1 > sweep_cap) { gr1e = o1 + sweep_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (flags) atomicOr(S.status, flags);
    dx[DX_SEND_L0] = o0; dx[DX_SEND_L1] = sl1; dx[DX_SEND_L1E] = sl1e;
    dx[DX_SEND_R0] = sr0; dx[DX_SEND_R1] = o1; dx[DX_SEND_R1B] = sr1b;
    dx[DX_GHOST_L0] = gl0; dx[DX_GHOST_L1] = o0; dx[DX_GHOST_L1B] = gl1b;
    dx[DX_GHOST_R0] = o1; dx[DX_GHOST_R1] = gr1; dx[DX_GHOST_R1E] = gr1e;
    int32_t *h = dx + DX_HDR_SEND;
    h[0] = sl1 - o0; h[1] = sl1e - o0; h[2] = sd[SD_STEP]; h[3] = 0;
    h[4] = o1 - sr0; h[5] = o1 - sr1b; h[6] = sd[SD_STEP]; h[7] = 0;
}

// Pack what goes to the neighbours (blockIdx.y = side: 0 = to the left, 1 = to the right) into the send staging:
// DX_ALIGN = the 4 records of the sgw boundary layers in this rank's sorted order, DX_VELD / DX_DFS / DX_ACC / DX_AUX /
// DX_MISC = one 16-byte word per particle of the outermost owned layer.  ctrl (may be NULL): a sweep behind the converged one has
// nothing new.
__global__ void k_dfsph_shard_pack(DevParams P, DevArrays S, const int32_t *dx, int what, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int side = blockIdx.y;
    const int b = side == 0 ? dx[DX_SEND_L0] : (what == DX_ALIGN ? dx[DX_SEND_R0] : dx[DX_SEND_R1B]);
    const int e = side == 0 ? (what == DX_ALIGN ? dx[DX_SEND_L1] : dx[DX_SEND_L1E]) : dx[DX_SEND_R1];
    if (s >= e - b) return;
    const int i = b + s;
    SPH_EMU_CHECK(s < P.halo_cap && i >= 0 && i < P.n);
    if (what == DX_ALIGN) {
        S.stage[side][0][s] = S.posm[i];
        S.stage[side][1][s] = S.veld[i];
        S.stage[side][2][s] = S.x0id[i];
        S.stage[side][3][s] = S.misc[i];
    } else {
        S.stage[side][0][s] = dx_sweep_array(S, what)[i];
    }
}

// Land what the neighbours sent on the ghost records (blockIdx.y = side: 0 = from the left, 1 = from the right).
// DX_ALIGN: rec[side][k] = the 4 arrays received; both ranks classified the same fp32 positions, so the sender's
// boundary layers and this rank's ghost layers hold the same records with the same per-cell counts and only the order
// inside a cell differs -- after the overwrite, ghost record begin + k IS the sender's boundary record k (cell_end stays
// valid).  A count mismatch leaves the ghost range alone and a record of another cell is not written; both set
// SPH_STATUS_GHOST_ALIGN.
// DX_VELD / DX_DFS / DX_ACC / DX_AUX: rec[side][0] = the words of the neighbour's outermost owned layer -> this rank's
// first ghost layer.  DX_MISC: only .y (the pressure) of each word -- misc.z carries FLAG_GHOST on this rank and not on
// the owner, and the alignment already brought the rest.
__global__ void k_dfsph_shard_unpack(DevParams P, DevArrays S, int32_t *dx, int what, const DfsphCtrl *ctrl,
                                     const float4 *rec00, const float4 *rec01, const float4 *rec02, const float4 *rec03,
                                     const float4 *rec10, const float4 *rec11, const float4 *rec12, const float4 *rec13) {
    if (ctrl && ctrl->done) return;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int side = blockIdx.y;
    if (side == 0 ? !P.has_left : !P.has_right) return;
    const int b = side == 0 ? (what == DX_ALIGN ? dx[DX_GHOST_L0] : dx[DX_GHOST_L1B]) : dx[DX_GHOST_R0];
    const int e = side == 0 ? dx[DX_GHOST_L1] : (what == DX_ALIGN ? dx[DX_GHOST_R1] : dx[DX_GHOST_R1E]);
    const float4 *r0 = side == 0 ? rec00 : rec10;
    if (what != DX_ALIGN) {
        if (s >= e - b) return;
        SPH_EMU_CHECK(s < P.halo_cap && b + s >= 0 && b + s < P.n);
        if (what == DX_MISC) S.misc[b + s].y = r0[s].y;
        else dx_sweep_array(S, what)[b + s] = r0[s];
        return;
    }
    const int32_t *h = dx + DX_HDR_RECV + 4 * side;
    const int first = side == 0 ? e - dx[DX_GHOST_L1B] : dx[DX_GHOST_R1E] - b;  // records of the first ghost layer
    if (h[0] != e - b || h[1] != first) {
        if (s == 0) atomicOr(S.status, SPH_STATUS_GHOST_ALIGN);
        return;
    }
    if (s >= e - b) return;
    const int g = b + s;
    SPH_EMU_CHECK(s < P.halo_cap && g >= 0 && g < P.n);
    const float4 p = r0[s], q = S.posm[g];
    int ci, cj, ck, di, dj, dk;
    const int c_new = cell_of(P, p.x, p.y, p.z, ci, cj, ck), c_old = cell_of(P, q.x, q.y, q.z, di, dj, dk);
    if (c_new != c_old) { atomicOr(S.status, SPH_STATUS_GHOST_ALIGN); return; }
    float4 m = side == 0 ? rec03[s] : rec13[s];
    m.z = __uint_as_float(__float_as_uint(m.z) | FLAG_GHOST);
    S.posm[g] = p;
    S.veld[g] = side == 0 ? rec01[s] : rec11[s];
    S.x0id[g] = side == 0 ? rec02[s] : rec12[s];
    S.misc[g] = m;
}
