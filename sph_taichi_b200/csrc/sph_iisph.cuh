// sph_iisph.cuh -- implicit incompressible SPH (reference IISPH.py, simulationMethod 3; Ihmsen et al. 2014) on top of
// the same sorted SoA state and per-step neighbour lists as the DFSPH path.
//
// The reference's IISPH.py cannot run (DESIGN section 10 lists why), so these kernels implement the formulation of
// DESIGN section 10 with its constants.  Per step: the DFSPH density pass (no clamp, no EOS; builds the lists),
// k_dfsph_non_pressure without cohesion, k_dfsph_predict_velocity (v* = v + dt a), k_iisph_predict (a_ii, s_i and
// the warm start), the relaxed Jacobi loop (k_iisph_pressure_accel<false> + k_iisph_pressure_update +
// k_iisph_check per sweep), k_iisph_pressure_accel<true> (final a^p + reactions on dynamic solids), k_iisph_advect.
// x-slab sharded (P.slab_on, sph_shard_iisph_step): every kernel but the density pass works on the owned records; the
// neighbours' values it reads in the first ghost layer -- v* in k_iisph_predict, aux.y = p / rho^2 in
// k_iisph_pressure_accel, acc = {a^p, 1} in k_iisph_pressure_update -- arrive with the exchanges of the outermost owned
// layer that the host issues after each kernel that changes them (DX_VELD, DX_AUX, DX_ACC).
// Sharded with dynamic solids (sph_shard_configure_iisph_bodies): compute_pressure_forces runs without the reaction
// scatter and k_iisph_shard_reactions gathers the same terms onto the owned dynamic solids, after one more exchange
// (DX_MISC) that brings the first ghost layer's final pressures.
//
// Per-step scratch, all in existing per-step workspace (no new sorted payload):
//   dfs[i]   = {a_ii, s_i, -, -}              (the DFSPH scratch; unused in an IISPH context)
//   acc[i]   = fluid after predict: {a^p_i, 1}  -- w = 1 marks a fluid a^p; solids keep {g or 0 (+ reactions), 0}
//   aux[i].y = fluid: p_i / rho_i^2             (the density pass leaves it 0 in DFSPH mode)
//   misc[i].y = p_i: the pressure record the sort carries, so the next step's warm start reads this step's result
// psi_j = rho0 * m_V_j is folded as rho0 * (sum over m_V_j ...) below.
#pragma once
#include "sph_dfsph.cuh"

enum IisphOp {
    IISPH_COMPUTE_DENSITIES = 0,         // compute_densities
    IISPH_NON_PRESSURE_FORCES = 1,       // compute_non_pressure_forces (gravity + viscosity)
    IISPH_PREDICT_ADVECTION = 2,         // predict_advection: v*, then a_ii, s_i and p = 0.5 p_prev
    IISPH_PRESSURE_SOLVE_ITERATION = 3,  // pressure_solve_iteration (arg = omega, out = double accumulator of the error)
    IISPH_PRESSURE_FORCES = 4,           // compute_pressure_forces (+ reactions on dynamic solids)
    IISPH_ADVECT = 5,                    // advect
};

// predict_advection, second pass (after k_dfsph_predict_velocity wrote v* into veld):
//   s_i  = rho0 - rho_i - dt * sum_{F+B} psi_j (v*_i - v*_j) . gradW_ij
//   a_ii = dt^2 [ G_i . c_i - (psi_i / rho_i^2) sum_F psi_j |gradW_ij|^2 ],  G_i = sum_{F+B} psi_j gradW_ij,
//   c_i  = -(1/rho_i^2) sum_F psi_j gradW_ij - (1/rho_i^2 + 1/rho0^2) sum_B psi_b gradW_ib
//   p_i <- 0.5 p_i (warm start from the previous step's pressure)
__global__ void __launch_bounds__(128) k_iisph_predict(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    const float4 pi = S.posm[i];
    const float4 vi = S.veld[i];
    float fx = 0.f, fy = 0.f, fz = 0.f, bx = 0.f, by = 0.f, bz = 0.f, sq = 0.f, div = 0.f;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        const float gs = gradw_of(P, r2);
        const float4 vj = __ldg(S.veld + j);
        div += pj.w * (((vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz) * gs);
        const float s = pj.w * gs;  // m_V_j gradW_ij = s * r
        if (__ldg(&S.aux[j].z) > 0.0f) {
            fx += s * rx; fy += s * ry; fz += s * rz;
            sq += pj.w * (gs * gs) * r2;
        } else {
            bx += s * rx; by += s * ry; bz += s * rz;
        }
    });
    const float rho = vi.w;
    const float inv_r2 = 1.0f / (rho * rho);
    const float cb = inv_r2 + P.inv_rho0sq;
    const float gx = fx + bx, gy = fy + by, gz = fz + bz;
    const float gc = -(gx * (inv_r2 * fx + cb * bx) + gy * (inv_r2 * fy + cb * by) + gz * (inv_r2 * fz + cb * bz));
    const float dt2r2 = P.dt * P.dt * P.rho0 * P.rho0;
    float4 d = S.dfs[i];
    d.x = dt2r2 * (gc - pi.w * inv_r2 * sq);
    d.y = P.rho0 - rho - P.dt * P.rho0 * div;
    S.dfs[i] = d;
    const float p = 0.5f * S.misc[i].y;
    S.misc[i].y = p;
    S.aux[i].y = p * inv_r2;
}

// a^p_i = -sum_F psi_j (p_i/rho_i^2 + p_j/rho_j^2) gradW_ij - sum_B psi_b (p_i/rho_i^2 + p_i/rho0^2) gradW_ib
// REACT = false: one sweep's first pass (ctrl: sph_iisph_solve's loop state, NULL from the op).
// REACT = true: compute_pressure_forces -- each dynamic solid neighbour b also receives
//   acc_b += -(rho_i / rho_b) (b's term of a^p_i), rho_b = the body density the density pass put in aux[b].x,
// the convention of k_dfsph_iteration<1>.
template <bool REACT>
__global__ void __launch_bounds__(128) k_iisph_pressure_accel(DevParams P, DevArrays S, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;  // a sweep launched behind the converged one
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    const float4 pi = S.posm[i];
    const float dpi = S.aux[i].y;
    const float dpb = dpi + S.misc[i].y * P.inv_rho0sq;
    const float f_react = REACT ? -S.veld[i].w : 0.0f;
    float ax = 0.f, ay = 0.f, az = 0.f;
    for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
        const float4 aj = __ldg(S.aux + j);
        const float gs = gradw_of(P, r2);
        if (aj.z > 0.0f) {
            const float c = pj.w * gs * (dpi + aj.y);
            ax -= c * rx; ay -= c * ry; az -= c * rz;
        } else {
            const float c = pj.w * gs * dpb;
            ax -= c * rx; ay -= c * ry; az -= c * rz;
            if (REACT && aj.z < -1.5f) {  // dynamic rigid body: reaction
                const float f = f_react / aj.x * P.rho0;
                float *a = reinterpret_cast<float *>(S.acc + j);
                atomicAdd(a + 0, -c * rx * f);
                atomicAdd(a + 1, -c * ry * f);
                atomicAdd(a + 2, -c * rz * f);
            }
        }
    });
    S.acc[i] = make_float4(P.rho0 * ax, P.rho0 * ay, P.rho0 * az, 1.0f);
}

// The reactions of compute_pressure_forces on the owned dynamic solids as a GATHER (sharded steps with dynamic solids;
// the counterpart of k_shard_reactions): the scatter of k_iisph_pressure_accel<true> would miss the fluid a neighbour
// owns across a cut.  One warp per solid id walks the 27 cells over the fluid records that hold this step's density
// and final pressure -- the owned layers and the first ghost layer, [SD_DENS0, SD_DENS1) -- with the neighbour lists'
// predicate (symmetric in i, b) and forms the solid branch of k_iisph_pressure_accel<true> operand for operand, so
// only the summation order differs from the single engine's float atomics.  What it reads from a ghost fluid record i
// and which message brought it: posm (alignment), veld.w = rho_i (DX_VELD, the owner's word), aux.y = p / rho^2 (the
// converged sweep's DX_AUX; aux.z > 0 marks a fluid), misc.y = p (DX_MISC).  acc[b] holds {g, 0} from
// k_dfsph_non_pressure; w stays 0.
__global__ void __launch_bounds__(128) k_iisph_shard_reactions(DevParams P, DevArrays S) {
    const int lane = threadIdx.x & 31;
    const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (s >= P.n_solid) return;  // warp-uniform
    const int b = S.solid_slot[s];
    if (!shard_owned_index(S, b)) return;
    if (!(__float_as_uint(S.misc[b].z) & FLAG_DYNAMIC)) return;
    const float4 pb = S.posm[b];
    const float rho_b = S.aux[b].x;  // the body density
    const int d0 = S.sd[SD_DENS0], d1 = S.sd[SD_DENS1];
    int ci, cj, ck;
    cell_of(P, pb.x, pb.y, pb.z, ci, cj, ck);
    ci = min(max(ci, 0), P.gx - 1); cj = min(max(cj, 0), P.gy - 1); ck = min(max(ck, 0), P.gz - 1);
    const int k_lo = max(ck - 1, 0), k_hi = min(ck + 1, P.gz - 1);
    float ax = 0.f, ay = 0.f, az = 0.f;
    for (int dx = -1; dx <= 1; ++dx) {
        int ni = ci + dx;
        if (ni < 0 || ni >= P.gx) continue;
        for (int dy = -1; dy <= 1; ++dy) {
            int nj = cj + dy;
            if (nj < 0 || nj >= P.gy) continue;
            int row = (ni * P.gy + nj) * P.gz;
            int i0 = max(__ldg(S.cell_end + max(row + k_lo - 1, 0)), d0);
            int i1 = min(__ldg(S.cell_end + row + k_hi), d1);
            for (int i = i0 + lane; i < i1; i += 32) {
                const float4 ai = __ldg(S.aux + i);
                if (!(ai.z > 0.0f)) continue;  // solid
                const float4 pi = __ldg(S.posm + i);
                float rx = pi.x - pb.x, ry = pi.y - pb.y, rz = pi.z - pb.z;
                if (!(exact_r2(rx, ry, rz) < P.h2)) continue;  // the density pass's list predicate
                const float gs = gradw_of(P, rx * rx + ry * ry + rz * rz);
                const float c = pb.w * gs * (ai.y + __ldg(&S.misc[i].y) * P.inv_rho0sq);
                const float f = -__ldg(&S.veld[i].w) / rho_b * P.rho0;
                ax += -c * rx * f; ay += -c * ry * f; az += -c * rz * f;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ax += __shfl_xor_sync(0xffffffffu, ax, o);
        ay += __shfl_xor_sync(0xffffffffu, ay, o);
        az += __shfl_xor_sync(0xffffffffu, az, o);
    }
    if (lane != 0) return;
    // the slot is read again rather than kept: with the divisions' slow-path calls in the loop, ptxas spilled it
    float4 *ab = S.acc + S.solid_slot[(blockIdx.x * blockDim.x + threadIdx.x) >> 5];
    float4 a = *ab;
    a.x += ax; a.y += ay; a.z += az;
    *ab = a;
}

// One sweep's second pass, with the sweep's error sum fused in (as k_dfsph_density_change_err):
//   (Ap)_i = dt^2 [ sum_F psi_j (a^p_i - a^p_j) . gradW_ij + sum_B psi_b a^p_i . gradW_ib ]
//   p_i <- max(p_i + omega (s_i - (Ap)_i) / a_ii, 0) if |a_ii| > 1e-6, else 0
//   err += |(Ap)_i - s_i| / rho0 over the fluid particles whose new p_i > 0
// acc[j].w is 1 for a fluid a^p and 0 for a solid, so one expression covers both kinds of neighbour.
__global__ void __launch_bounds__(128) k_iisph_pressure_update(DevParams P, DevArrays S, float omega, double *err_out,
                                                               const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;  // written only by k_iisph_check, between kernels: uniform over the grid
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    double e = 0.0;
    if (dfsph_fluid(P, S, i, fl)) {
        const float4 pi = S.posm[i];
        const float4 api = S.acc[i];
        float ap = 0.f;
        for_listed_neighbors(P, S, i, pi, [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
            const float4 aj = __ldg(S.acc + j);
            const float gs = gradw_of(P, r2);
            ap += pj.w * gs * ((api.x - aj.w * aj.x) * rx + (api.y - aj.w * aj.y) * ry + (api.z - aj.w * aj.z) * rz);
        });
        ap *= P.dt * P.dt * P.rho0;
        const float2 d = *reinterpret_cast<const float2 *>(S.dfs + i);  // {a_ii, s_i}
        float p = 0.0f;
        if (fabsf(d.x) > 1e-6f) p = fmaxf(S.misc[i].y + omega * (d.y - ap) / d.x, 0.0f);
        S.misc[i].y = p;
        const float rho = S.veld[i].w;
        S.aux[i].y = p / (rho * rho);
        if (p > 0.0f) e = (double)(fabsf(ap - d.y) / P.rho0);
    }
    dfsph_block_sum_to<4>(e, err_out);
}

// The loop of pressure_solve, evaluated on the device after every sweep:
//   it = 0;  while it < max_iterations:  avg = sweep() / n_fluid;  it += 1;  if avg < eta: break
// err is the sweep's whole error sum (this rank's, or the rank-ordered sum of all ranks' partials).
__device__ __forceinline__ void iisph_check_sum(DfsphCtrl *ctrl, double err, double n_fluid, double eta,
                                                int32_t max_iterations) {
    const double avg = err / n_fluid;
    ctrl->last_avg = avg;
    ctrl->err = 0.0;
    ctrl->sweeps += 1;
    ctrl->iterations = ctrl->sweeps;
    if (avg < eta || ctrl->sweeps >= max_iterations) ctrl->done = 1;
}
__global__ void k_iisph_check(DfsphCtrl *ctrl, double n_fluid, double eta, int32_t max_iterations) {
    if (ctrl->done) return;
    iisph_check_sum(ctrl, ctrl->err, n_fluid, eta, max_iterations);
}
// Sharded: parts = the all-gathered error partials, added in rank order (ranked_err_sum), so every rank takes the same
// decision after the same sweep.
__global__ void k_iisph_check_ranked(DfsphCtrl *ctrl, const double *parts, int32_t rank, int32_t world, double n_fluid,
                                     double eta, int32_t max_iterations) {
    if (ctrl->done) return;
    iisph_check_sum(ctrl, ranked_err_sum(ctrl, parts, rank, world), n_fluid, eta, max_iterations);
}

// advect: v += dt * acc, x += dt * v for every dynamic particle -- the fluid's acc holds a^p and its veld v*, so this
// is v = v* + dt a^p; a dynamic solid integrates g + reactions as k_dfsph_advect does.  Sharded: a particle that moves
// a whole cell layer in x in one step is flagged (SPH_STATUS_SHARD_VELOCITY), as in k_dfsph_advect.
__global__ void k_iisph_advect(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!dfsph_in_range(P, S, i)) return;
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i];
    const float4 a = S.acc[i];
    v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    S.veld[i] = v;
    if (P.slab_on && !(fabsf(v.x) * P.dt < P.h)) atomicOr(S.status, SPH_STATUS_SHARD_VELOCITY);
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    S.posm[i] = p;
}

// sph_iisph_read: a_ii, s_i and a^p in the current (sorted) order; 0 for solids
__global__ void k_iisph_read(DevParams P, DevArrays S, float *a_ii, float *s, float *ap) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const bool fluid = (__float_as_uint(S.misc[i].z) & FLAG_FLUID) != 0;
    const float4 d = S.dfs[i], a = S.acc[i];
    if (a_ii) a_ii[i] = fluid ? d.x : 0.0f;
    if (s) s[i] = fluid ? d.y : 0.0f;
    if (ap) {
        ap[3 * i] = fluid ? a.x : 0.0f;
        ap[3 * i + 1] = fluid ? a.y : 0.0f;
        ap[3 * i + 2] = fluid ? a.z : 0.0f;
    }
}
