// sph_common.cuh -- shared device-side types and math for libsph_b200 (sm_90a).
//
// Data layout in HBM (all arrays sorted by flattened cell id, z fastest, like the reference's
// counting sort; particle_system.py:292-294,322-369).  Everything a pair kernel gathers per
// neighbour is one aligned 16-byte word, so a gather is a single LDG.128/LDS.128:
//   posm[i] = {x, y, z, m_V}                         (particle_system.py:103,107)
//   veld[i] = {vx, vy, vz, density}                  (particle_system.py:105,109)
//   aux[i]  = fluid: {m/rho_unclamped, p/rho^2, m, 0}   solid: {body density, 0, -1|-2, 0}
//             (-1 static, -2 dynamic) -- per-step derived data written by the density pass
//   x0id[i] = {x_0, y_0, z_0, object_id bits}        (particle_system.py:102,104)
//   misc[i] = {m, pressure, flags bits, solid_id bits}
//             flags = material | is_dynamic << 1 | color r,g,b << 8,16,24
//   acc[i]  = {ax, ay, az, 0}                        (particle_system.py:106)
#pragma once
#ifdef SPH_EMU  // host-side emulation of the kernel source (tests/emu/): stand-ins for CUDA and the PTX helpers
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#include "sph_ptx.cuh"
#endif
#include <stdint.h>

#include <cmath>

// Invariants the kernels state about their own index arithmetic.  They compile to nothing in the product; the
// host-side emulation build (tests/emu/cuda_emu.h) turns them into aborting checks.
#ifndef SPH_EMU_CHECK
#define SPH_EMU_CHECK(cond) ((void)0)
#endif

#include "../../include/sph_b200.h"

#define FLAG_FLUID 1u
#define FLAG_DYNAMIC 2u
#define FLAG_GHOST 4u  // x-slab sharding: copy of a neighbour rank's particle, never integrated

struct DevParams {
    int32_t n;
    int32_t n_solid;
    int32_t C;
    int32_t gx, gy, gz;
    float h, h2, h2_scan, inv_h, d2;  // h2: r2 < h2 <=> sqrtf(r2) < h exactly; h2_scan: conservative prefilter
    float m_V0, rho0, inv_rho0sq, stiffness, exponent;
    int32_t exponent_int;  // >0: exponent is that small integer (multiply chain), else powf
    float sigma, d_visc, visc_eps, dt;
    float gx_, gy_, gz_;
    float k_w, k2_w, k_dw, w0, w_diam;
    float k1_grad, wd_norm;  // 6k / h and W(diameter) / 2k: normalisations of spline_pair()
    float pad, hi_x, hi_y, hi_z;
    // x-slab sharding (multi-GPU, sph_shard_*): this rank keeps sgw ghost layers per side; the slab [sx0, sx1)
    // itself, the live count and the send / receive ranges live in DEVICE memory (DevArrays::sd) so that a whole
    // sharded step -- sort, pair passes and halo exchange -- replays from one CUDA graph without the host.
    // In this mode n is the CAPACITY of the arrays; the last 2 * halo_cap records are the receive regions
    // (left neighbour, then right neighbour).
    int32_t slab_on, sgw, halo_cap, has_left, has_right, rebalance_every;
    // all fluid particles share one mass and one volume (true for every scene the reference can
    // express with a single fluid density): the force pass then needs only 2 x 16 B per neighbour
    int32_t uniform_fluid;
    float fluid_m, fluid_mV;
    int32_t dfsph;  // simulationMethod 4: the density pass neither clamps nor evaluates the EOS
    int32_t opaque_zero;  // always 0; lets a kernel state a scheduling dependency ptxas cannot fold away
    // nibble p = the (dx, dy) column c = (dx + 1) * 3 + (dy + 1) the density pass visits p-th.  The list order is
    // free (only the summation order of the pair passes depends on it); centre column first makes the lanes of
    // a warp gather the SAME records at the same time in the force pass
    unsigned long long col_order;
};

struct DevArrays {
    float4 *posm, *veld, *x0id, *misc, *acc;       // current (sorted) state
    float4 *posm_n, *veld_n, *x0id_n, *misc_n, *acc_n;  // sort destination
    float4 *aux;
    // per-step packed neighbour records of the uniform-fluid force pass (written by the density pass),
    // 32 bytes per particle so that ONE 256-bit load (LDG.E.256) gathers a neighbour:
    //   fpv[2i]     = {x, y, z, fluid: m/rho_unclamped | solid: m_V}
    //   fpv[2i + 1] = {vx, vy, vz, fluid: p/rho^2 (>= 0) | solid: -body density (dynamic) or -inf (static)}
    float4 *fpv;
    float4 *dfs;  // DFSPH: {dfsph_factor, density_adv, -, -} (particle_system.py:115-117)
    int32_t *cid;       // cell id per particle in pre-sort order
    int32_t *grid_ids;  // cell id per particle in sorted order (public grid_ids)
    int32_t *perm;      // bucket slot -> pre-sort index
    int32_t *cell_end;  // [C] inclusive prefix sum (public grid_particles_num)
    int32_t *ticket;    // arrival ticket of each particle inside its cell (from the histogram atomic)
    unsigned long long *tile_state;
    int32_t *tile_counter;
    int32_t *solid_slot;  // [n_solid] solid_id -> sorted index
    uint32_t *status;
    // per-step neighbour lists, built by the density pass and re-used by the force pass:
    // nbr_list[k * npad + i] = sorted index of the k-th neighbour of particle i (k < NBR_CAP),
    // in the reference's visiting order; nbr_cnt[i] = count, or NBR_OVERFLOW.
    int32_t *nbr_list;
    int32_t *nbr_cnt;
    int32_t npad;
    // x-slab sharding: device-resident step state (SD_* below) and the send staging of the two sides
    // (0 = to the left neighbour, 1 = to the right): 4 record arrays of halo_cap entries + a 16-int header
    int32_t *sd;
    float4 *stage[2][4];
    int32_t *stage_hdr[2];
};

// DevArrays::sd (ints).  Header layout (sent with every exchange): {records, owned, sx0, sx1, step}.
enum {
    SD_N_LIVE = 0,   // sorted records [0, n_live) are owned or ghost; [n_live, n_sorted) is the trash bucket
    SD_OWNED, SD_SX0, SD_SX1, SD_STEP,
    SD_OWN0, SD_OWN1,                            // index range of the owned cell layers
    SD_SEND_L0, SD_SEND_L1, SD_SEND_R0, SD_SEND_R1,  // index ranges packed for the left / right neighbour
    SD_RECV_L, SD_RECV_R,                        // records received for THIS step's classification
    SD_N_SORTED, SD_FLAGS, SD_DENS0,                   // [DENS0, DENS1): index range that needs densities
    // (DENS1 follows the headers)
    SD_HDR_L = 16, SD_HDR_R = 32,                // headers received from the left / right neighbour
    SD_SENT_LO = 48, SD_SENT_HI,                 // records sent so far (64-bit, for the halo statistics)
    SD_DENS1 = 50,
    SD_DB_L1 = 51, SD_DB_R0 = 52,                // boundary density ranges: [DENS0, DB_L1) and [DB_R0, DENS1)
    SD_INTS = 64
};
constexpr int SHARD_MIN_WIDTH = 5;  // a slab gives a layer away only while it is wider than this (ghost band 2 + send range 4 must fit)

// Sharded steps replay from a CUDA graph, so their grids are fixed while the record counts are device state:
// the light kernels run grid-stride loops over a COMPACT input numbering -- u in [0, n_live + recv_l + recv_r) --
// instead of launching one (mostly idle) thread per slot of the capacity.
__device__ __forceinline__ int shard_input_total(const int32_t *__restrict__ sd) {
    return sd[SD_N_LIVE] + sd[SD_RECV_L] + sd[SD_RECV_R];
}
__device__ __forceinline__ int shard_input_index(const DevParams &P, const int32_t *__restrict__ sd, int u) {
    const int nl = sd[SD_N_LIVE], cl = sd[SD_RECV_L];
    if (u < nl) return u;
    if (u < nl + cl) return P.n - 2 * P.halo_cap + (u - nl);
    return P.n - P.halo_cap + (u - nl - cl);
}


constexpr int NBR_CAP = 96;  // soak runs of the shipped scenes peak at 54 neighbours (tools/soak.py)
constexpr int NBR_OVERFLOW = 0x7fffffff;
#ifndef LIST_PAD_VALUE
#define LIST_PAD_VALUE 4
#endif
constexpr int LIST_PAD = LIST_PAD_VALUE;  // lists are padded with the particle's own index to a multiple of this

// |r|^2 in the reference's (and the oracle's) rounding sequence: three products, two sums, no FMA
// contraction.  With P.h2 this makes the neighbour predicate `(x_i - x_j).norm() < h`
// (particle_system.py:384) bit-exact, which matters on lattices where many pairs sit at r == h and
// DFSPH counts neighbours (DFSPH.py:171-176).
__device__ __forceinline__ float exact_r2(float rx, float ry, float rz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry)), __fmul_rn(rz, rz));
}

// r = sqrt(r2) and 1/r from one MUFU.RSQ (|rel err| ~ 1e-7); exact 0 for coincident particles
__device__ __forceinline__ void fast_norm(float r2, float &r, float &inv_r) {
    float t = rsqrt_ftz(r2);
    inv_r = (r2 > 0.0f) ? t : 0.0f;
    r = r2 * inv_r;
}

// Branch-free cubic spline (sph_base.py:23-68) in the two-sided form
//     W(q) = 2k (a^3 - 4 b^3),   dW/dq = 6k (4 b^2 - a^2),   a = max(1 - q, 0), b = max(1/2 - q, 0),
// algebraically identical to the reference's piecewise polynomials (q <= 1/2: k(6q^3 - 6q^2 + 1) and
// 6k q(3q - 2)); rounding differs by a few ulp of W(0).  Returns wn = W / (2k) and G with
// grad W = (6k / h) * G * r_vec.  The reference's `r > 1e-5` guard on the gradient is applied to r^2;
// below it r is treated as 0 (W(1e-5) and W(0) differ by 4e-7 relative).
__device__ __forceinline__ void spline_pair(const DevParams &P, float r2, float &wn, float &G) {
    float t = rsqrt_ftz(r2);
    float inv_r = (r2 > 1e-10f) ? t : 0.0f;
    float r = r2 * inv_r;
    float a = fmaf(-r, P.inv_h, 1.0f);
    float b = fmaxf(a - 0.5f, 0.0f);
    a = fmaxf(a, 0.0f);
    float a2 = a * a, b2 = b * b;
    G = fmaf(4.0f, b2, -a2) * inv_r;
    wn = fmaf(b2 * b, -4.0f, a2 * a);
}
// density-only variant: W / (2k)
__device__ __forceinline__ float spline_w_norm(const DevParams &P, float r2) {
    float r = r2 * rsqrt_ftz(fmaxf(r2, 1e-30f));  // exact 0 for coincident particles
    float a = fmaf(-r, P.inv_h, 1.0f);
    float b = fmaxf(a - 0.5f, 0.0f);
    a = fmaxf(a, 0.0f);
    return fmaf(b * b * b, -4.0f, a * a * a);
}

// grad W = s * r_vec, division-free variant of gradw_scale()
__device__ __forceinline__ float gradw_scale_fast(const DevParams &P, float r, float inv_r) {
    float q = r * P.inv_h;
    float f = 1.0f - q;
    float s = (q <= 0.5f) ? P.k_dw * q * (3.0f * q - 2.0f) : P.k_dw * (-f * f);
    return (r > 1e-5f && q <= 1.0f) ? s * (inv_r * P.inv_h) : 0.0f;
}

__device__ __forceinline__ int cell_of(const DevParams &P, float x, float y, float z, int &ci, int &cj, int &ck) {
    // particle_system.py:287-294 -- true division by the f32 grid size, truncation toward zero
    ci = (int)(x / P.h);
    cj = (int)(y / P.h);
    ck = (int)(z / P.h);
    return ci * P.gy * P.gz + cj * P.gz + ck;
}

// sph_base.py:23-44
__device__ __forceinline__ float w_cubic(const DevParams &P, float r) {
    float q = r * P.inv_h;
    float res;
    if (q <= 0.5f) {
        float q2 = q * q;
        res = P.k_w * (6.0f * q2 * q - 6.0f * q2 + 1.0f);
    } else {
        float f = fmaxf(1.0f - q, 0.0f);
        res = P.k2_w * (f * f * f);
    }
    return res;
}

// sph_base.py:46-68: returns s such that grad W = s * r_vec  (r = |r_vec| < h assumed)
__device__ __forceinline__ float gradw_scale(const DevParams &P, float r) {
    float q = r * P.inv_h;
    float s;
    if (q <= 0.5f) {
        s = P.k_dw * q * (3.0f * q - 2.0f);
    } else {
        float f = 1.0f - q;
        s = P.k_dw * (-f * f);
    }
    return (r > 1e-5f && q <= 1.0f) ? s / (r * P.h) : 0.0f;
}

__device__ __forceinline__ float tait_pressure(const DevParams &P, float rho_clamped) {
    // WCSPH.py:76
    float x = rho_clamped / P.rho0;
    float pw;
    if (P.exponent_int == 7) {
        float x2 = x * x, x4 = x2 * x2;
        pw = x4 * x2 * x;
    } else if (P.exponent_int > 0) {
        pw = 1.0f;
        for (int e = 0; e < P.exponent_int; ++e) pw *= x;
    } else {
        pw = powf(x, P.exponent);
    }
    return P.stiffness * (pw - 1.0f);
}

// Walk the 27-cell neighbourhood in the reference's order (x offset slowest, z fastest;
// particle_system.py:378-385).  For fixed (dx, dy) the three z-cells are contiguous in the
// sorted arrays, so the walk is 9 contiguous index ranges.  Cells outside the grid are skipped
// (SURVEY Q3); cell 0 is invisible exactly as in the reference (Q2) because a range always
// starts at cell_end[max(c - 1, 0)].  fn(j, rx, ry, rz, r2, posm_j) is called for j != i, r2 < h2.
template <int STRIDE = 1, typename F>
__device__ __forceinline__ void for_all_neighbors(const DevParams &P, const float4 *__restrict__ posm,
                                                  const int32_t *__restrict__ cell_end, int i, float xi, float yi,
                                                  float zi, F &&fn) {
    int ci, cj, ck;
    cell_of(P, xi, yi, zi, ci, cj, ck);
    int k_lo = max(ck - 1, 0), k_hi = min(ck + 1, P.gz - 1);
    for (int dx = -1; dx <= 1; ++dx) {
        int ni = ci + dx;
        if (ni < 0 || ni >= P.gx) continue;
        for (int dy = -1; dy <= 1; ++dy) {
            int nj = cj + dy;
            if (nj < 0 || nj >= P.gy) continue;
            int row = (ni * P.gy + nj) * P.gz;
            int c_lo = row + k_lo, c_hi = row + k_hi;
            int j0 = __ldg(cell_end + max(c_lo - 1, 0));
            int j1 = __ldg(cell_end + c_hi);
            for (int j = j0; j < j1; ++j) {
                float4 pj = __ldg(posm + (size_t)j * STRIDE);
                float rx = xi - pj.x, ry = yi - pj.y, rz = zi - pj.z;
                float r2 = exact_r2(rx, ry, rz);
                if (r2 < P.h2 && j != i) fn(j, rx, ry, rz, r2, pj);
            }
        }
    }
}

// Host side: every derived constant the kernels read (particle_system.py:38,43-46; sph_base.py:23-68).
inline void derive_dev_params(DevParams &P, const SphParams &h) {
    P.gx = h.grid_num[0]; P.gy = h.grid_num[1]; P.gz = h.grid_num[2];
    P.C = P.gx * P.gy * P.gz;
    P.h = h.h; P.inv_h = 1.0f / h.h; P.d2 = h.diameter * h.diameter;
    {   // h2 = min{t : sqrtf(t) >= h}: then r2 < h2 <=> sqrtf(r2) < h, the reference's predicate, exactly
        float t = h.h * h.h;
        while (std::sqrt(t) >= h.h) t = std::nextafter(t, 0.0f);
        while (std::sqrt(std::nextafter(t, INFINITY)) < h.h) t = std::nextafter(t, INFINITY);
        P.h2 = std::nextafter(t, INFINITY);
        P.h2_scan = P.h2 * 1.000002f;  // FFMA-chain prefilter: a superset of the exact hits
    }
    P.m_V0 = h.m_V0; P.rho0 = h.density0; P.inv_rho0sq = 1.0f / (h.density0 * h.density0);
    P.stiffness = h.stiffness; P.exponent = h.exponent;
    float er = std::round(h.exponent);
    P.exponent_int = (er == h.exponent && er >= 1.f && er <= 16.f) ? (int)er : 0;
    P.sigma = h.surface_tension; P.d_visc = (float)(2.0 * (3 + 2) * (double)h.viscosity);
    P.visc_eps = h.visc_eps; P.dt = h.dt;
    P.gx_ = h.g[0]; P.gy_ = h.g[1]; P.gz_ = h.g[2];
    P.k_w = h.k_w; P.k2_w = h.k_w * 2.0f; P.k_dw = h.k_dw; P.w0 = h.k_w;
    {   // W(d) on the host with the same expression the device uses
        float q = h.diameter * P.inv_h;
        if (q <= 0.5f) { float q2 = q * q; P.w_diam = h.k_w * (6.0f * q2 * q - 6.0f * q2 + 1.0f); }
        else { float f = 1.0f - q; if (f < 0) f = 0; P.w_diam = P.k2_w * (f * f * f); }
    }
    P.k1_grad = P.k_dw * P.inv_h; P.wd_norm = P.w_diam / P.k2_w;
    P.opaque_zero = 0;
    if (P.col_order == 0ull) P.col_order = 0x862075314ull;  // centre, edges, corners (4 1 3 5 7 0 2 6 8)
    P.pad = h.h; P.hi_x = h.clamp_hi[0]; P.hi_y = h.clamp_hi[1]; P.hi_z = h.clamp_hi[2];
}
