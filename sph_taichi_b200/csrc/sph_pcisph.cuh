// sph_pcisph.cuh -- predictive-corrective incompressible SPH (simulationMethod 1; Solenthaler & Pajarola 2009, the
// reference's legacy engine/sph_solver.py pci_* methods) on top of the same sorted SoA state and per-step neighbour
// lists as the DFSPH path.
//
// The legacy PCISPH is 2-D code with a racy error estimate, so these kernels implement the 3-D formulation of DESIGN
// section 11 with its constants.  Per step: the DFSPH density pass (no clamp, no EOS; builds the lists at x^t),
// k_dfsph_non_pressure without cohesion + k_pcisph_init (pci_compute_deltas: a^np, p = 0, a^p = 0), the
// prediction-correction loop (k_pcisph_predict + k_pcisph_update_pressure + k_pcisph_pressure_force<false> +
// k_pcisph_check per sweep), k_pcisph_pressure_force<true> (the final a^p + reactions on dynamic solids),
// k_pcisph_advect (pci_update_time_step).
// x-slab sharded (P.slab_on, sph_shard_pcisph_step; fluid and static solids): every kernel but the density pass works on
// the owned records.  What a sweep reads of the first ghost layer arrives with the exchanges of the outermost owned
// layer that the host issues after the kernel that changes it: dfs = {x*, m_V} after k_pcisph_predict (DX_DFS; a
// solid's word is the x^t k_pcisph_init set) and misc.y = p after k_pcisph_update_pressure (DX_MISC).  Nothing else of
// a ghost is read after the alignment -- the first sweep's pressure update reads no neighbour p, and the final pressure
// force reads the last sweep's words -- so no once-per-step message precedes the loop.  The sweep's error is the max
// over the ranks' fp64 partials (k_pcisph_check_ranked).
//
// Per-step scratch, all in existing per-step workspace (no new sorted payload):
//   acc[i]    = {a^np_i, 0}: gravity + viscosity (fluid); g or 0 (+ reactions) for a solid
//   dfs[i]    = {x*_i, m_V_i}: the predicted position (fluid; a solid keeps x^t) and the volume -- the record a
//               neighbour gathers in both list walks of a sweep
//   aux[i]    = fluid after k_pcisph_init: {a^p_i, rho*_i}  (a solid keeps the density pass's {rho_b, 0, -1|-2, 0})
//   misc[i].y = p_i, with the flags in misc.z: the second record the pressure force gathers
//   veld[i]   = {v^t_i, rho_i} until k_pcisph_advect
// So the predicted density gathers ONE 16-byte word per neighbour (dfs) and the pressure force two (dfs, misc); the
// reaction of the final pass also reads veld[b].w = rho_b of a dynamic solid neighbour.  The 27-cell fallback of an
// overflowed list adds posm (the predicate at x^t).
#pragma once
#include "sph_dfsph.cuh"

enum PcisphOp {
    PCISPH_COMPUTE_DENSITIES = 0,        // compute_densities (also builds the neighbour lists)
    PCISPH_COMPUTE_DELTAS = 1,           // pci_compute_deltas: a^np (gravity + viscosity), p = 0, a^p = 0
    PCISPH_POS_VEL_PREDICTION = 2,       // pci_pos_vel_prediction: v*, x*
    PCISPH_UPDATE_PRESSURE = 3,          // pci_update_pressure (arg = delta, out = int32 max of the error's bits)
    PCISPH_UPDATE_PRESSURE_FORCE = 4,    // pci_update_pressure_force: a^p at x*
    PCISPH_COMPUTE_PRESSURE_FORCES = 5,  // compute_pressure_forces: the same a^p + reactions on dynamic solids
    PCISPH_UPDATE_TIME_STEP = 6,         // pci_update_time_step
};

// Walk over the step's neighbour list of fluid particle i (the density pass's order, built at x^t), gathering each
// neighbour's predicted record dfs[j] = {x*_j, m_V_j} instead of its position; falls back to the 27-cell scan at x^t
// when the list overflowed.  fn(j, rec_j).
template <typename F>
__device__ __forceinline__ void pcisph_for_listed(const DevParams &P, const DevArrays &S, int i, F &&fn) {
    const int cnt = S.nbr_cnt[i];
    if (cnt != NBR_OVERFLOW) {
        const int32_t *lp = S.nbr_list + i;
        const size_t stride = (size_t)S.npad;
        for (int k0 = 0; k0 < cnt; k0 += 4) {
            int j[4];
            float4 rj[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                j[u] = (k0 + u < cnt) ? lp[(size_t)(k0 + u) * stride] : i;
                rj[u] = __ldg(S.dfs + j[u]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (k0 + u < cnt) fn(j[u], rj[u]);
        }
    } else {
        const float4 pi = S.posm[i];
        for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z,
                          [&](int j, float, float, float, float, const float4 &) { fn(j, __ldg(S.dfs + j)); });
    }
}

// r = x*_i - x*_j and |r|^2 with one fixed rounding sequence (every kernel below forms it the same way)
__device__ __forceinline__ float pcisph_r(const float4 &xi, const float4 &xj, float &rx, float &ry, float &rz) {
    rx = xi.x - xj.x; ry = xi.y - xj.y; rz = xi.z - xj.z;
    return fmaf(rx, rx, fmaf(ry, ry, __fmul_rn(rz, rz)));
}

// grad W(x*_i - x*_j) = gs * r: gradw_of's spline, written with explicit roundings only (products and sums that the
// compiler may not contract), so that both instantiations of k_pcisph_pressure_force compute the same bits
__device__ __forceinline__ float pcisph_gradw(const DevParams &P, float r2) {
    float r, inv_r;
    fast_norm(r2, r, inv_r);
    const float q = __fmul_rn(r, P.inv_h);
    const float f = __fadd_rn(1.0f, -q);
    const float s = (q <= 0.5f) ? __fmul_rn(__fmul_rn(P.k_dw, q), fmaf(3.0f, q, -2.0f))
                                : __fmul_rn(P.k_dw, -__fmul_rn(f, f));
    return (r > 1e-5f && q <= 1.0f) ? __fmul_rn(s, __fmul_rn(inv_r, P.inv_h)) : 0.0f;
}

// pci_compute_deltas, second half (after k_dfsph_non_pressure wrote a^np into acc): p = 0, a^p = 0, rho* = 0 and the
// predicted record of every particle = its position (a solid's stays so for the whole loop)
__global__ void k_pcisph_init(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!dfsph_in_range(P, S, i)) return;
    S.dfs[i] = S.posm[i];
    if (!(__float_as_uint(S.misc[i].z) & FLAG_FLUID)) return;
    S.misc[i].y = 0.0f;
    S.aux[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// v* = v + dt (a^np + a^p), x* = x + dt v*: the expression of the prediction and of pci_update_time_step
__device__ __forceinline__ float4 pcisph_velocity(const DevParams &P, const float4 &v, const float4 &anp, const float4 &ap) {
    return make_float4(fmaf(P.dt, anp.x + ap.x, v.x), fmaf(P.dt, anp.y + ap.y, v.y), fmaf(P.dt, anp.z + ap.z, v.z), v.w);
}

// a. pci_pos_vel_prediction (fluid only; ctrl: sph_pcisph_solve's loop state, NULL from the op)
__global__ void k_pcisph_predict(DevParams P, DevArrays S, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;  // a sweep launched behind the converged one
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    const float4 x = S.posm[i];
    const float4 v = pcisph_velocity(P, S.veld[i], S.acc[i], S.aux[i]);
    S.dfs[i] = make_float4(fmaf(P.dt, v.x, x.x), fmaf(P.dt, v.y, x.y), fmaf(P.dt, v.z, x.z), x.w);
}

// This rank's error max as an fp64 partial: the bits of the exactly converted double, maxed as an unsigned integer
// (non-negative doubles order as their bits, a NaN's above every number), so the partial is exact and independent of
// order.  m = a warp's max of the float bits.
__device__ __forceinline__ void pcisph_max_partial(double *part, int32_t m) {
    const double e = (double)__int_as_float(m);
#ifdef SPH_EMU  // the host emulation has no 64-bit atomicMax
    uint64_t b, *u = reinterpret_cast<uint64_t *>(part);
    std::memcpy(&b, &e, 8);
    uint64_t old = __atomic_load_n(u, __ATOMIC_SEQ_CST);
    while (old < b && !__atomic_compare_exchange_n(u, &old, b, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
#else
    atomicMax(reinterpret_cast<unsigned long long *>(part), (unsigned long long)__double_as_longlong(e));
#endif
}

// b. pci_update_pressure, with the sweep's error max fused in:
//   rho*_i = rho0 (m_V_i W(0) + sum_{F+B} m_V_j W(x*_i - x*_j)),  e_i = max(rho*_i - rho0, 0),  p_i <- p_i + delta e_i
//   err_max = max_i e_i as the int bits of the non-negative float (exact, independent of order)
// err_part (sharded loops; NULL otherwise): the same max as this rank's fp64 partial (pcisph_max_partial)
__global__ void __launch_bounds__(128) k_pcisph_update_pressure(DevParams P, DevArrays S, float delta, int32_t *err_max,
                                                                double *err_part, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;  // written only by k_pcisph_check, between kernels: uniform over the grid
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    float e = 0.0f;
    if (dfsph_fluid(P, S, i, fl)) {
        const float4 xi = S.dfs[i];
        float den = 0.0f;
        pcisph_for_listed(P, S, i, [&](int, const float4 &xj) {
            float rx, ry, rz;
            den = fmaf(xj.w, spline_w_norm(P, pcisph_r(xi, xj, rx, ry, rz)), den);
        });
        const float rho = fmaf(den, P.k2_w, xi.w * P.w0) * P.rho0;
        const float d = rho - P.rho0;
        e = !(d <= 0.0f) ? d : 0.0f;  // a NaN stays a NaN (and stops nothing)
        S.misc[i].y = fmaf(delta, e, S.misc[i].y);
        S.aux[i].w = rho;
    }
    const int m = __reduce_max_sync(0xffffffffu, __float_as_int(e));
    if ((threadIdx.x & 31) == 0 && m > 0) {
        atomicMax(err_max, m);
        if (err_part) pcisph_max_partial(err_part, m);
    }
}

// c. pci_update_pressure_force (REACT = false) and compute_pressure_forces (REACT = true):
//   a^p_i = -sum_F psi_j (p_i + p_j) / rho0^2 gradW(x*_i - x*_j) - sum_B psi_b 2 p_i / rho0^2 gradW(x*_i - x_b)
// psi_j = rho0 m_V_j, so a^p = -(1/rho0) sum m_V_j (p_i + p_j or 2 p_i) gradW.  REACT also gives each dynamic solid
// neighbour b the reaction acc_b += -(rho_i / rho_b) (b's term of a^p_i), rho_b = veld[b].w, the convention of
// k_iisph_pressure_accel<true>; a^p comes out bit-identical to REACT = false (every rounding of a^p is explicit).
template <bool REACT>
__global__ void __launch_bounds__(128) k_pcisph_pressure_force(DevParams P, DevArrays S, const DfsphCtrl *ctrl) {
    if (ctrl && ctrl->done) return;
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t fl;
    if (!dfsph_fluid(P, S, i, fl)) return;
    const float4 xi = S.dfs[i];
    const float pi = S.misc[i].y;
    const float inv_rho0 = 1.0f / P.rho0;
    const float f_react = REACT ? S.veld[i].w * inv_rho0 : 0.0f;
    float ax = 0.f, ay = 0.f, az = 0.f;
    pcisph_for_listed(P, S, i, [&](int j, const float4 &xj) {
        const float4 mj = __ldg(S.misc + j);
        const uint32_t flj = __float_as_uint(mj.z);
        float rx, ry, rz;
        const float gs = pcisph_gradw(P, pcisph_r(xi, xj, rx, ry, rz));
        const float c = __fmul_rn(__fmul_rn(xj.w, gs), __fadd_rn(pi, (flj & FLAG_FLUID) ? mj.y : pi));
        ax = fmaf(-c, rx, ax); ay = fmaf(-c, ry, ay); az = fmaf(-c, rz, az);
        if (REACT && (flj & (FLAG_FLUID | FLAG_DYNAMIC)) == FLAG_DYNAMIC) {  // dynamic rigid body: reaction
            const float f = f_react / __ldg(&S.veld[j].w);
            float *a = reinterpret_cast<float *>(S.acc + j);
            atomicAdd(a + 0, __fmul_rn(__fmul_rn(c, rx), f));
            atomicAdd(a + 1, __fmul_rn(__fmul_rn(c, ry), f));
            atomicAdd(a + 2, __fmul_rn(__fmul_rn(c, rz), f));
        }
    });
    float4 a = S.aux[i];
    a.x = __fmul_rn(ax, inv_rho0); a.y = __fmul_rn(ay, inv_rho0); a.z = __fmul_rn(az, inv_rho0);
    S.aux[i] = a;
}

// The loop of the prediction-correction step, evaluated on the device after every sweep:
//   it = 0;  do { sweep();  it += 1 } while (!((err < eta rho0 and it >= min_iterations) or it >= max_iterations))
// threshold = eta rho0 in fp64; err = the sweep's max error, last_avg keeps it.
__device__ __forceinline__ void pcisph_check_max(DfsphCtrl *ctrl, double err, double threshold, int32_t min_iterations,
                                                 int32_t max_iterations) {
    ctrl->last_avg = err;
    ctrl->err_max = 0;
    ctrl->sweeps += 1;
    ctrl->iterations = ctrl->sweeps;
    if ((err < threshold && ctrl->sweeps >= min_iterations) || ctrl->sweeps >= max_iterations) ctrl->done = 1;
}
__global__ void k_pcisph_check(DfsphCtrl *ctrl, double threshold, int32_t min_iterations, int32_t max_iterations) {
    if (ctrl->done) return;
    pcisph_check_max(ctrl, (double)__int_as_float(ctrl->err_max), threshold, min_iterations, max_iterations);
}
// Sharded: parts = the all-gathered fp64 partials of the other ranks, this rank's own still in ctrl->err.  Their max
// (a NaN in any of them wins, as in the integer max of one rank) is exact and does not depend on the order, so every
// rank takes the same decision after the same sweep and keeps the same last_avg bits.
__global__ void k_pcisph_check_ranked(DfsphCtrl *ctrl, const double *parts, int32_t rank, int32_t world,
                                      double threshold, int32_t min_iterations, int32_t max_iterations) {
    if (ctrl->done) return;
    double err = ctrl->err;
    for (int r = 0; r < world; ++r)
        if (r != rank && !(err != err || parts[r] <= err)) err = parts[r];
    ctrl->err = 0.0;
    pcisph_check_max(ctrl, err, threshold, min_iterations, max_iterations);
}

// pci_update_time_step: fluid v = v + dt (a^np + a^p), x = x + dt v with the final a^p; a dynamic solid integrates
// g + reactions as k_dfsph_advect does.  Sharded: a particle that moves a whole cell layer in x in one step is flagged
// (SPH_STATUS_SHARD_VELOCITY), as in k_dfsph_advect.
__global__ void k_pcisph_advect(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!dfsph_in_range(P, S, i)) return;
    const uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i];
    const float4 a = S.acc[i];
    if (fl & FLAG_FLUID) {
        v = pcisph_velocity(P, v, a, S.aux[i]);
    } else {
        v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    }
    S.veld[i] = v;
    if (P.slab_on && !(fabsf(v.x) * P.dt < P.h)) atomicOr(S.status, SPH_STATUS_SHARD_VELOCITY);
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    S.posm[i] = p;
}

// sph_pcisph_read: rho*, p and a^p in the current (sorted) order; 0 for solids
__global__ void k_pcisph_read(DevParams P, DevArrays S, float *rho_star, float *p, float *ap) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const bool fluid = (__float_as_uint(S.misc[i].z) & FLAG_FLUID) != 0;
    const float4 a = S.aux[i];
    if (rho_star) rho_star[i] = fluid ? a.w : 0.0f;
    if (p) p[i] = fluid ? S.misc[i].y : 0.0f;
    if (ap) {
        ap[3 * i] = fluid ? a.x : 0.0f;
        ap[3 * i + 1] = fluid ? a.y : 0.0f;
        ap[3 * i + 2] = fluid ? a.z : 0.0f;
    }
}
