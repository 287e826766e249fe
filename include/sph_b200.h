/*
 * sph_b200.h -- C ABI of libsph_b200.so, the sm_90a (H100) WCSPH step engine.
 *
 * The reference (erizmr/SPH_Taichi @ 4a701fd) is pure Python + Taichi and has NO FFI of its
 * own: the drop-in boundary is the Python class surface ParticleSystem / SPHBase /
 * WCSPHSolver (SURVEY.md section 8b).  This ABI sits directly underneath that surface; each
 * entry point names the reference method(s) (file:line) whose device work it replaces.  The
 * Python shells in sph_taichi_b200/ bind it with ctypes (see INTEGRATION.md for the binding a
 * reference maintainer would add).
 *
 * Conventions
 *   - every function returns 0 on success, a negative SPH_E_* code on failure; the message
 *     is available from sph_last_error().  No C++ exceptions cross the ABI.
 *   - all device work is enqueued asynchronously on the cudaStream_t passed as `stream`
 *     (a `void*`; NULL = legacy default stream).  No hidden synchronisation except where
 *     stated (sph_read_status, sph_get_timers).
 *   - device memory is owned by the caller (PyTorch): the caller allocates one workspace of
 *     sph_workspace_bytes() bytes and the public per-particle arrays; the context only
 *     carves the workspace.  One context per GPU / process; not thread-safe.
 *   - there is no CPU fallback: every entry point fails with SPH_E_CUDA if no device work
 *     can be launched.
 */
#ifndef SPH_B200_H
#define SPH_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPH_OK 0
#define SPH_E_ARG (-1)      /* bad argument / state */
#define SPH_E_CUDA (-2)     /* CUDA runtime error */
#define SPH_E_CAPACITY (-3) /* workspace too small / too many particles */
#define SPH_E_NCCL (-4)

#define SPH_MATERIAL_SOLID 0 /* particle_system.py:30 */
#define SPH_MATERIAL_FLUID 1 /* particle_system.py:31 */

/* device status word bits (sph_read_status) */
#define SPH_STATUS_OUT_OF_GRID 1u /* a particle hashed outside the grid (reference: OOB write) */
#define SPH_STATUS_BAD_POLAR 2u   /* shape matching hit a singular A */
#define SPH_STATUS_HALO_CAPACITY 4u  /* sharded: a send range exceeded halo_capacity (records were cut off) */
#define SPH_STATUS_SHARD_CAPACITY 8u /* sharded: live + received records ran into the receive regions */
#define SPH_STATUS_SHARD_VELOCITY 16u /* sharded DFSPH: a particle moved >= one cell layer in x in one step */
#define SPH_STATUS_GHOST_ALIGN 32u   /* sharded DFSPH: a neighbour's boundary layers and the ghost layers differ */
#define SPH_STATUS_SOLID_SLOT 64u    /* sharded with dynamic solids: two live records carry the same solid id */

/* Scalar parameters.  All constants are folded in double on the host exactly as the
 * reference folds them in Python scope before Taichi bakes them into kernels
 * (particle_system.py:33-46, sph_base.py:11-21,23-68, WCSPH.py:8-16). */
typedef struct SphParams {
    int32_t dim;            /* must be 3 (2-D is unreachable in the reference, SURVEY section 2) */
    int32_t grid_num[3];    /* ceil(domain_size / h)                   particle_system.py:44 */
    float h;                /* support radius = grid size = padding     particle_system.py:37,43,46 */
    float diameter;         /* particle diameter                        particle_system.py:36 */
    float m_V0;             /* 0.8 d^3                                  particle_system.py:38 */
    float density0;         /*                                          sph_base.py:17-18 */
    float stiffness;        /*                                          WCSPH.py:12-13 */
    float exponent;         /*                                          WCSPH.py:9-10 */
    float viscosity;        /* 0.01                                     sph_base.py:15 */
    float surface_tension;  /* 0.01                                     WCSPH.py:15 */
    float dt;               /*                                          WCSPH.py:16 */
    float g[3];             /*                                          sph_base.py:13 */
    float domain_size[3];   /* domainEnd - domainStart                  particle_system.py:22 */
    float k_w;              /* 8 / (pi h^3)                             sph_base.py:27-35 */
    float k_dw;             /* 6 * k_w                                  sph_base.py:50-58 */
    float visc_eps;         /* 0.01 h^2                                 WCSPH.py:113 */
    float clamp_hi[3];      /* domain_size - padding                    sph_base.py:155-173 */
} SphParams;

/* Public per-particle arrays in the reference's field layout (particle_system.py:102-140):
 * 3-vectors are AoS [n][3].  Pointers are DEVICE pointers.  `solid_id` is an extra i32 array
 * prepared by the host shell: a dense immutable id 0..n_solid-1 for solid particles (the
 * particles of one object contiguous), -1 for fluid; may be NULL when there are no solids. */
typedef struct SphFields {
    int32_t *object_id;
    float *x, *x_0, *v, *acceleration;
    float *m_V, *m, *density, *pressure;
    int32_t *material, *is_dynamic;
    int32_t *color;    /* [n][3], each component must be in 0..255 */
    int32_t *grid_ids; /* output only (particle_system.py:138) */
    int32_t *solid_id; /* input only */
    float *dfsph_factor, *density_adv; /* DFSPH, output only, may be NULL (particle_system.py:115-117) */
} SphFields;

/* One dynamic rigid body registered for shape matching (sph_base.py:200-260). */
typedef struct SphRigidBody {
    int32_t object_id;
    int32_t solid_begin, solid_end; /* range of solid_id values owned by this body */
    float rest_cm[3];               /* rest centre of mass (rigid_rest_cm, sph_base.py:87-89); NaN until computed */
} SphRigidBody;

typedef struct SphCtx SphCtx;

/* ---- lifetime ------------------------------------------------------------------------ */
/* Workspace bytes needed for n_max particles, n_solid solid particles, n_bodies bodies.
 * Capacity: 96 * round_up(n_max, 32) < 2^32 (per-step neighbour lists use 32-bit slots), i.e. n_max <= 44.7 M
 * particles per GPU; sph_create returns SPH_E_CAPACITY beyond that (shard by x-slabs, sph_shard_*). */
uint64_t sph_workspace_bytes(const SphParams *params, int64_t n_max, int64_t n_solid, int32_t n_bodies);
int sph_create(const SphParams *params, int64_t n_max, int64_t n_solid, int32_t n_bodies, int32_t device,
               void *workspace, uint64_t workspace_bytes, SphCtx **out);
int sph_destroy(SphCtx *ctx);
const char *sph_last_error(const SphCtx *ctx); /* ctx may be NULL: last creation error */
int sph_set_params(SphCtx *ctx, const SphParams *params); /* e.g. solver.dt[None] = ...; grid must not change */

/* ---- state transfer: ParticleSystem fields <-> packed sorted SoA (particle_system.py:102-140, 409-418) -- */
/* number of solid particles among the n packed ones (<= n_solid of sph_create) and whether any
 * of them is dynamic; call before sph_pack. */
int sph_set_solid_count(SphCtx *ctx, int64_t n_solid, int32_t has_dynamic_solids);
/* hint: every fluid particle has mass fluid_m and volume fluid_mV (lets the force pass gather 32
 * instead of 48 bytes per neighbour); uniform = 0 selects the general kernels. Call before sph_pack. */
int sph_set_fluid_uniform(SphCtx *ctx, int32_t uniform, float fluid_m, float fluid_mV);
int sph_pack(SphCtx *ctx, const SphFields *fields, int64_t n, void *stream);
int sph_unpack(SphCtx *ctx, const SphFields *fields, void *stream);
int sph_unpack_xv(SphCtx *ctx, float *x, float *v, int32_t *object_id, void *stream); /* dump(): particle_system.py:409-418 */
int sph_upload_xv(SphCtx *ctx, const float *x, const float *v, void *stream);         /* overwrite x, v in current order */
/* inclusive cell prefix sums, the reference's grid_particles_num after the scan (particle_system.py:374) */
int sph_copy_grid_particles_num(SphCtx *ctx, int32_t *out_dev, void *stream);

/* ---- the hot path, one entry per reference method ----------------------------------------- */
/* ParticleSystem.initialize_particle_system: update_grid_id + prefix sum + counting_sort
 * (particle_system.py:311-375; scan_single_buffer.py:108-146) */
int sph_neighbor_build(SphCtx *ctx, void *stream);
/* SPHBase.compute_static_boundary_volume (moving=0) / compute_moving_boundary_volume (moving=1)
 * (sph_base.py:91-113) */
int sph_boundary_volume(SphCtx *ctx, int32_t moving, void *stream);
/* WCSPHSolver.compute_densities (WCSPH.py:33-43) */
int sph_compute_densities(SphCtx *ctx, void *stream);
/* WCSPHSolver.compute_non_pressure_forces (WCSPH.py:128-140) */
int sph_compute_non_pressure_forces(SphCtx *ctx, void *stream);
/* WCSPHSolver.compute_pressure_forces (WCSPH.py:70-85) */
int sph_compute_pressure_forces(SphCtx *ctx, void *stream);
/* WCSPHSolver.advect (WCSPH.py:143-149) */
int sph_advect(SphCtx *ctx, void *stream);
/* SPHBase.enforce_boundary_3D(particle_type) (sph_base.py:149-179) */
int sph_enforce_boundary(SphCtx *ctx, int32_t particle_type, void *stream);

/* ---- rigid bodies (sph_base.py:182-260) --------------------------------------------------- */
int sph_set_rigid_bodies(SphCtx *ctx, const SphRigidBody *bodies, int32_t n_bodies);
/* compute_com (sph_base.py:182-192): centre of mass of body `index` -> out_dev[3] */
int sph_compute_com(SphCtx *ctx, int32_t body_index, float *out_dev, void *stream);
/* compute_rigid_rest_cm (sph_base.py:87-89): store current CoM as the rest CoM */
int sph_compute_rigid_rest_cm(SphCtx *ctx, int32_t body_index, void *stream);
/* solve_constraints (sph_base.py:200-222): shape matching; R (row-major 3x3) -> R_out_dev (may be NULL) */
int sph_solve_constraints(SphCtx *ctx, int32_t body_index, float *R_out_dev, void *stream);
/* R (row-major 3x3) and centre of mass of the body's last solve (also inside sph_step): 12 floats;
 * what the reference returns to the host for the OBJ export (sph_base.py:251-257) */
int sph_get_rigid_state(SphCtx *ctx, int32_t body_index, float *out_dev12, void *stream);

/* ---- SPHBase.step (sph_base.py:263-271) + WCSPHSolver.substep (WCSPH.py:152-156) ---------- */
/* nsteps whole steps with the fused kernels, replayed from a CUDA graph. */
int sph_step(SphCtx *ctx, int32_t nsteps, void *stream);

/* ---- DFSPH (reference DFSPH.py, simulationMethod 4; SURVEY.md section 8f rank 1) ---------------------
 * One entry point, `op` selects the reference kernel (names as in DFSPH.py):
 *   0 compute_densities (:39-47; also builds the neighbour lists)   1 compute_DFSPH_factor (:114-139)
 *   2 compute_density_change (:157-178)   3 compute_density_adv (:198-205)
 *   4 compute_density_error (:221-227; arg = offset, out_dev = zero-initialised double accumulator)
 *   5 multiply_time_step(dfsph_factor, arg) (:229-233)
 *   6 divergence_solver_iteration_kernel (:278-290)   7 pressure_solve_iteration_kernel (:354-367)
 *   8 compute_non_pressure_forces (:92-101)   9 predict_velocity (:392-397)   10 advect (:104-111)
 * With these ops the convergence loops (divergence_solve, pressure_solve) run on the host, as in the reference.
 * sph_set_dfsph(1) switches the density pass to DFSPH semantics (no clamp, no EOS). */
int sph_set_dfsph(SphCtx *ctx, int32_t enable);
int sph_dfsph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream);
/* The Jacobi loop of divergence_solve (mode 0, DFSPH.py:245-254: sweeps of op 6 + op 2 + op 4 with offset 0) or of
 * pressure_solve (mode 1, DFSPH.py:323-331: op 7 + op 3 + op 4 with offset density_0) with the loop condition
 *     while m < 1 or m < max_iterations:  avg = sweep() / n_fluid;  if avg <= eta: break;  m += 1
 * evaluated on the device after every sweep.  Sweeps are launched `first_batch` at a time (then in pairs); sweeps
 * behind the converged one return immediately; the host waits once per batch instead of once per sweep.  The
 * steps the reference performs before and after the loop (ops 2 / 3 and 5) stay with the caller.  SYNCHRONOUS:
 * returns m (iterations_out), the sweeps executed and the last avg (host pointers, may be NULL). */
int sph_dfsph_solve(SphCtx *ctx, int32_t mode, int32_t max_iterations, double eta, float offset, int64_t n_fluid,
                    int32_t first_batch, int32_t *iterations_out, int32_t *sweeps_out, double *avg_err_out,
                    void *stream);

/* One whole SPHBase.step() of the DFSPH solver (sph_base.py:263-271 with DFSPH.substep, DFSPH.py:399-408): neighbour
 * build, moving boundary volumes, compute_densities, compute_DFSPH_factor, divergence_solve (if enabled),
 * compute_non_pressure_forces, predict_velocity, pressure_solve, advect, solve_rigid_body, enforce_boundary_3D(fluid)
 * -- every kernel launched from this one call, the two Jacobi loops run as in sph_dfsph_solve.  A DFSPH step is
 * ~50 launches; issuing them all from C++ keeps the Python host loop out of the way (the step is then bound by its
 * Jacobi sweeps).  The caller fills the constants exactly as the reference's host code computes them. */
typedef struct SphDfsphStep {
    int32_t enable_divergence_solver;   /* DFSPH.py:12 */
    int32_t max_iterations_v, max_iterations; /* m_max_iterations_v, m_max_iterations */
    double eta_v, eta;                  /* 1/dt * max_error_V * 0.01 * density_0 ; max_error * 0.01 * density_0 */
    float inv_dt, dt, inv_dt2;          /* the three factors multiply_time_step is called with (DFSPH.py:240, 262, 320) */
    float density0;                     /* offset of the pressure loop's density error (DFSPH.py:317) */
    int64_t n_fluid;                    /* fluid_particle_num (the error sums are averaged over it) */
    int32_t first_batch_v, first_batch; /* in: sweeps launched before the first wait; out: sweeps the last step's loops ran */
    int32_t iterations_v, iterations;   /* out: m_iterations_v, m_iterations of the last step */
    double avg_err_v, avg_err;          /* out: the last avg_density_err of each loop */
} SphDfsphStep;
int sph_dfsph_step(SphCtx *ctx, int32_t nsteps, SphDfsphStep *io, void *stream);

/* ---- IISPH (implicit incompressible SPH, reference IISPH.py, simulationMethod 3) -------------------------------
 * The reference's IISPH.py cannot run; these calls implement the formulation DESIGN.md section 10 states (its
 * deviations from IISPH.py are listed there).  sph_set_iisph(1) puts a context in IISPH mode: the density pass has
 * DFSPH semantics (no clamp, no EOS), and the WCSPH / DFSPH calls (sph_step, sph_dfsph_*, sph_shard_step,
 * sph_shard_profile_step, sph_shard_dfsph_step) and sph_shard_configure_bodies refuse the context (dynamic solids in
 * IISPH shard through sph_shard_configure_iisph_bodies only); sph_set_dfsph or sph_set_iisph(0) leave the mode (the context is then a WCSPH one unless
 * sph_set_dfsph(1) follows; sph_set_iisph(0) on a context that is not in IISPH mode changes nothing).  An IISPH context
 * may be x-slab sharded: sph_set_iisph(1) BEFORE sph_shard_configure (it is refused on a sharded context), then
 * sph_shard_iisph_step (below).  The IISPH calls refuse a context that is not in IISPH mode, and sph_iisph_op,
 * sph_iisph_solve and sph_iisph_step refuse a sharded one (their grids cover the capacity, ghosts and trash included).
 * One op per reference method (IISPH.py names):
 *   0 compute_densities (also builds the neighbour lists)   1 compute_non_pressure_forces (gravity + viscosity)
 *   2 predict_advection (v* = v + dt a; a_ii, s_i; p = 0.5 p_prev)
 *   3 pressure_solve_iteration (arg = omega; out_dev = zero-initialised double accumulator of sum |Ap - s| / rho0)
 *   4 compute_pressure_forces (a^p with the final pressures + reactions on dynamic solids)   5 advect */
int sph_set_iisph(SphCtx *ctx, int32_t enable);
int sph_iisph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream);
/* pressure_solve's relaxed Jacobi loop
 *     it = 0;  while it < max_iterations:  avg = sweep() / n_fluid;  it += 1;  if avg < eta: break
 * with the loop condition evaluated on the device after every sweep (batches of sweeps as in sph_dfsph_solve; the
 * first batch is first_batch sweeps).  SYNCHRONOUS: returns it and the last avg (host pointers, may be NULL). */
int sph_iisph_solve(SphCtx *ctx, int32_t max_iterations, float omega, double eta, int64_t n_fluid, int32_t first_batch,
                    int32_t *iterations_out, double *avg_err_out, void *stream);
/* nsteps whole IISPH SPHBase.step()s: neighbour build, moving boundary volumes, ops 0-2, the loop of sph_iisph_solve,
 * ops 4-5, solve_rigid_body, enforce_boundary_3D(fluid) -- every kernel launched from this one call. */
typedef struct SphIisphStep {
    int32_t max_iterations; /* 1000 */
    float omega;            /* relaxation, 0.5 */
    double eta;             /* the loop stops when the average error < eta (1e-3) */
    int64_t n_fluid;        /* fluid particles (the error sum is averaged over them) */
    int32_t first_batch;    /* in: sweeps launched before the first wait; out: sweeps the last step ran */
    int32_t iterations;     /* out: sweeps of the last step's loop */
    double avg_err;         /* out: its last average error */
} SphIisphStep;
int sph_iisph_step(SphCtx *ctx, int32_t nsteps, SphIisphStep *io, void *stream);
/* Per-step scratch of the last IISPH kernels, in the current (sorted) order of sph_unpack: a_ii [n], s_i [n] and the
 * pressure acceleration a^p [n][3] (device pointers, each may be NULL; 0 for solids).  a^p is the last sweep's until
 * op 4 replaces it with the final one. */
int sph_iisph_read(SphCtx *ctx, float *a_ii, float *s, float *ap, void *stream);

/* ---- PCISPH (predictive-corrective incompressible SPH, simulationMethod 1; the legacy engine's pci_* methods) ----
 * These calls implement the 3-D formulation DESIGN.md section 11 states (its deviations from the legacy 2-D code are
 * listed there).  sph_set_pcisph(1) puts a context in PCISPH mode: the density pass has DFSPH semantics (no clamp, no
 * EOS), and the WCSPH, DFSPH and IISPH calls (sph_step, sph_dfsph_*, sph_iisph_*, sph_shard_step,
 * sph_shard_profile_step, sph_shard_dfsph_step, sph_shard_iisph_step), sph_shard_configure and the body configures
 * refuse the context.  A PCISPH context may be x-slab sharded (fluid + static solids): sph_set_pcisph(1) BEFORE
 * sph_shard_configure_pcisph (it is refused on a sharded context), then sph_shard_pcisph_step (below).  sph_set_dfsph,
 * sph_set_iisph(1) or sph_set_pcisph(0) leave the mode (sph_set_pcisph(0) on a context that is not in PCISPH mode
 * changes nothing).  The PCISPH calls refuse a context that is not in PCISPH mode, and sph_pcisph_op, sph_pcisph_solve
 * and sph_pcisph_step refuse a sharded one (their grids cover the capacity, ghosts and trash included).  One op per
 * method name:
 *   0 compute_densities (also builds the neighbour lists)
 *   1 pci_compute_deltas (a^np = gravity + viscosity; p = 0, a^p = 0)
 *   2 pci_pos_vel_prediction (v* = v + dt (a^np + a^p), x* = x + dt v*; solids stay at x^t)
 *   3 pci_update_pressure (arg = delta; out_dev = zero-initialised int32 that receives the max of the sweep's error
 *     max(rho* - rho0, 0) as the bits of a float)
 *   4 pci_update_pressure_force (a^p at x*)
 *   5 compute_pressure_forces (the same a^p + reactions on dynamic solids)   6 pci_update_time_step */
int sph_set_pcisph(SphCtx *ctx, int32_t enable);
int sph_pcisph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream);
/* The prediction-correction loop (ops 2-4 per sweep)
 *     it = 0;  do { sweep();  it += 1 } while (!((max_err < eta rho0 and it >= min_iterations) or it >= max_iterations))
 * with the loop condition evaluated on the device after every sweep (batches of sweeps as in sph_dfsph_solve; the
 * first batch is first_batch sweeps).  SYNCHRONOUS: returns it and the last max error (host pointers, may be NULL). */
int sph_pcisph_solve(SphCtx *ctx, float delta, double eta, int32_t min_iterations, int32_t max_iterations,
                     int32_t first_batch, int32_t *iterations_out, double *max_err_out, void *stream);
/* nsteps whole PCISPH SPHBase.step()s: neighbour build, moving boundary volumes, ops 0-1, the loop of sph_pcisph_solve,
 * ops 5-6, solve_rigid_body, enforce_boundary_3D(fluid) -- every kernel launched from this one call. */
typedef struct SphPcisphStep {
    float delta;            /* pressure per unit of density error (pci_scaling_factor; fp64 on the host, rounded) */
    double eta;             /* the loop may stop once the max density error < eta rho0 (0.01) */
    int32_t min_iterations; /* 3 */
    int32_t max_iterations; /* 1000 */
    int32_t first_batch;    /* in: sweeps launched before the first wait; out: sweeps the last step ran */
    int32_t iterations;     /* out: sweeps of the last step's loop */
    double max_err;         /* out: the last sweep's max density error (kg/m^3) */
} SphPcisphStep;
int sph_pcisph_step(SphCtx *ctx, int32_t nsteps, SphPcisphStep *io, void *stream);
/* Per-step scratch of the last PCISPH kernels, in the current (sorted) order of sph_unpack: the predicted density
 * rho* [n], the pressure p [n] and the pressure acceleration a^p [n][3] (device pointers, each may be NULL; 0 for
 * solids). */
int sph_pcisph_read(SphCtx *ctx, float *rho_star, float *p, float *ap, void *stream);

/* ---- x-slab sharding across the GPUs of one node (new; the reference is single-device) -------
 * One process per GPU.  Each rank owns the cell layers [x_lo, x_hi) of the x axis (x-major flattening,
 * particle_system.py:292-294: after the sort every layer is ONE contiguous index range) and keeps
 * `ghost_layers` (2) layers of copies of its neighbours' particles, so ONE exchange per step suffices.
 * Everything a step needs lives on the device -- live count, slab bounds, send / receive ranges, record counts
 * (carried in-band in a header) -- so a whole sharded step is a fixed launch sequence (capturable as ONE CUDA graph):
 *
 *     plan (receive counts, cut re-balancing) -> classify + sort -> info (send ranges) -> densities within one
 *     layer of the send ranges -> forces + integration of the send ranges, written straight into the send staging
 *     -> { halo exchange of the NEXT step  ||  interior densities -> staged state back into the arrays -> interior
 *     forces + integration }
 *
 * and the host only launches.  Every record is classified as owned / ghost / dropped from its position
 * alone (both ranks evaluate the same fp32 expression), so migration needs no extra message; cuts move by at
 * most one layer every `rebalance_every` steps, decided identically on both sides of a cut from the owned
 * counts in the headers.  Scenes with one fluid (uniform masses) and any number of STATIC solids: a solid record
 * rides the exchange like a fluid one (posm.w = its boundary volume m_V, misc = material, flags, solid_id) and is
 * staged unchanged, so the caller must pack every solid with its final start-up m_V -- the value the single engine's
 * sph_boundary_volume computes over the WHOLE scene (a solid's neighbours may sit across a cut).  Dynamic solids
 * (shape-matched bodies, advected rigid blocks) shard only through sph_shard_configure_bodies (WCSPH) and
 * sph_shard_configure_iisph_bodies (IISPH), both below; in DFSPH they are single-GPU.  sph_shard_configure refuses them, and on a sharded
 * context sph_set_solid_count refuses the dynamic flag, sph_set_rigid_bodies a body table, and sph_boundary_volume,
 * sph_compute_com, sph_compute_rigid_rest_cm and sph_solve_constraints refuse to run (they walk solid ids through a
 * slot map that migration leaves stale for solids of other ranks).
 *
 * DFSPH contexts (sph_set_dfsph(1) before sph_shard_configure) step with sph_shard_dfsph_step instead: the same
 * classification, sort, re-balancing and end-of-step record exchange, plus a once-per-step ghost alignment (each
 * rank overwrites its ghost layers with the neighbour's owned boundary layers in the neighbour's sorted order) and
 * small exchanges of the outermost owned layer's velocities / {factor, density_adv} whenever the owner changes them
 * -- two per Jacobi sweep.  The loops' error sums are all-gathered and added in rank order, so every rank takes the
 * same convergence decision and issues the same transport calls.
 *
 * IISPH contexts (sph_set_iisph(1) before sph_shard_configure; fluid + static solids) step with sph_shard_iisph_step:
 * the same step shape as sph_shard_dfsph_step, with the outermost owned layer's v* sent after predict_velocity, its
 * aux word (p / rho^2) after the diagonal / source pass and after every pressure update, and its acc word (a^p) after
 * every pressure-acceleration pass -- two exchanges per relaxed Jacobi sweep.  With dynamic solids
 * (sph_shard_configure_iisph_bodies) one more word follows the loop: the final pressures (misc.y).
 *
 * PCISPH contexts (sph_set_pcisph(1), then sph_shard_configure_pcisph; fluid + static solids) step with
 * sph_shard_pcisph_step: the same step shape, with the outermost owned layer's predicted record {x*, m_V} sent after
 * every prediction and its pressure (misc.y) after every pressure update -- two exchanges per prediction-correction
 * sweep, and none outside the loop.
 *
 * The exchange goes through an SphTransport: NCCL point-to-point (libnccl.so.2 is dlopen'ed; the communicator
 * belongs to this library, created from an id the caller distributes), or caller-supplied functions (the CPU
 * test-suite routes them to torch.distributed / gloo against the host-emulated build); set it before
 * sph_shard_configure. */
typedef struct SphTransport {
    void *user;
    int (*group_start)(void *user);
    int (*group_end)(void *user, void *stream);
    int (*send)(void *user, const void *buf, uint64_t bytes, int32_t peer, void *stream);
    int (*recv)(void *user, void *buf, uint64_t bytes, int32_t peer, void *stream);
} SphTransport;
int sph_comm_unique_id(char out128[128]);                                  /* ncclGetUniqueId (rank 0) */
int sph_comm_init_nccl(SphCtx *ctx, const char id128[128], int32_t rank, int32_t world); /* ncclCommInitRank */
int sph_comm_set_transport(SphCtx *ctx, const SphTransport *t, int32_t rank, int32_t world);
/* The context must have been created with n_max = the per-rank CAPACITY (owned + ghosts + trash + 2 *
 * halo_capacity receive slots) and packed with this rank's initial particles.  halo_capacity = records per
 * side and direction (>= (ghost_layers + 2) fullest layers). */
int sph_shard_configure(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                        int32_t rebalance_every);
/* Opt-in sharding of WCSPH scenes with DYNAMIC solids: shape-matched bodies (`bodies`, solid-id ranges of the WHOLE
 * scene's ids, rest_cm computed over the whole scene; n_bodies = 0: advected rigid blocks only) and advected rigid
 * blocks.  Pack first (sph_set_solid_count with the whole scene's solid count and the dynamic flag, uniform fluid);
 * needs ghost_layers >= 3 (a moving solid's m_V in the second ghost layer sums solids of the third).  DFSPH contexts
 * are refused.  sph_shard_step then runs, eagerly on `stream` (no overlap, SPH_SHARD_GRAPH does not apply):
 *     plan -> sort -> info -> solid-id slot map of the live records (SPH_STATUS_SOLID_SLOT on a duplicate id)
 *     -> moving boundary volumes of the owned layers and ghost layers 1-2 -> densities -> forces + integration of
 *     the owned fluid -> the fluid's reactions GATHERED onto each owned dynamic solid (fluid of the owned layers and
 *     ghost layer 1) + its advection -> {x, m} and x_0 of the owned body particles -> all-gather of those records
 *     (one transport group, (world - 1) * 32 bytes per body particle sent) -> sph_step's shape matching (the same
 *     fp32 reduction in the same order) on every rank, and clamps -> the record exchange.
 * cm and R are bit-identical on every rank (sph_get_rigid_state works on every rank) and equal to the single
 * engine's for the same particle positions; ghost copies catch up through the record exchange.  The body table is fixed: sph_set_rigid_bodies, the per-body calls, sph_boundary_volume,
 * sph_shard_profile_step and sph_shard_dfsph_step are refused on such a context. */
int sph_shard_configure_bodies(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                               int32_t rebalance_every, const SphRigidBody *bodies, int32_t n_bodies);
/* Opt-in sharding of IISPH scenes with DYNAMIC solids: the arguments, checks and layout of sph_shard_configure_bodies
 * (ghost_layers >= 3, the whole scene's body table with rest_cm), on a context in IISPH mode -- sph_set_iisph(1) must
 * have been called before it; WCSPH and DFSPH contexts are refused.  IISPH scatters the rigid reactions once per step,
 * after the pressure loop, so no per-sweep reaction exchange is needed.  sph_shard_iisph_step then runs
 *     plan -> classify + sort -> info -> DX ranges -> ghost alignment (3 layers) -> solid-id slot map -> moving
 *     boundary volumes (owned layers + ghost layers 1-2) -> the IISPH substep of sph_shard_iisph_step, whose final
 *     pressure acceleration does NOT scatter reactions -> [misc: the final pressures] -> the reactions GATHERED onto
 *     each owned dynamic solid (fluid of the owned layers and ghost layer 1) -> advect -> body records -> all-gather
 *     -> shape matching on every rank, and clamps -> fluid wall clamp -> the record exchange.
 * Only the summation order of the reactions differs from sph_iisph_step.  cm and R are bit-identical on every rank.
 * Transport groups per step: alignment, v*, warm-start aux, two per sweep launched, the final pressures, the body
 * all-gather (world > 1 and a non-empty body table), the record exchange.  The refusals of a
 * sph_shard_configure_bodies context apply (body table fixed, solid-id calls, sph_shard_step, sph_shard_profile_step,
 * sph_shard_dfsph_step, the single-GPU IISPH calls). */
int sph_shard_configure_iisph_bodies(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers,
                                     int64_t halo_capacity, int32_t rebalance_every, const SphRigidBody *bodies,
                                     int32_t n_bodies);
/* Opt-in sharding of PCISPH scenes: the arguments, checks and layout of sph_shard_configure, on a context in PCISPH mode
 * -- sph_set_pcisph(1) must have been called before it; WCSPH, DFSPH and IISPH contexts are refused (they use
 * sph_shard_configure), and so is a context with dynamic solids (dynamic solids in PCISPH are single-GPU).  The context
 * then steps with sph_shard_pcisph_step; sph_shard_begin, sph_shard_info and sph_shard_dump work on it as on the others. */
int sph_shard_configure_pcisph(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                               int32_t rebalance_every);
/* first sort of the packed particles + the first halo exchange (no physics) */
int sph_shard_begin(SphCtx *ctx, void *stream);
/* nsteps sharded SPHBase.step()s (sph_base.py:263-271): asynchronous launches that run ahead of the device (no host
 * synchronisation inside a step); SPH_SHARD_GRAPH=1 replays one captured CUDA graph per step instead */
int sph_shard_step(SphCtx *ctx, int32_t nsteps, void *stream);
/* nsteps sharded DFSPH SPHBase.step()s (sph_base.py:263-271 with DFSPH.substep, DFSPH.py:399-408) of a DFSPH context
 * (fluid + static solids): the step of sph_dfsph_step with `io` used the same way, except that io->n_fluid is the GLOBAL fluid
 * count (all ranks).  Every rank returns the same iterations, first_batch and avg_err values.  Eager launches with
 * one host wait per batch of Jacobi sweeps, like sph_dfsph_step (SPH_SHARD_GRAPH does not apply).  A particle that
 * moves a whole cell layer in x in one step sets SPH_STATUS_SHARD_VELOCITY (the record exchange would lose it);
 * sph_shard_info reports the status word. */
int sph_shard_dfsph_step(SphCtx *ctx, int32_t nsteps, SphDfsphStep *io, void *stream);
/* nsteps sharded IISPH SPHBase.step()s of an IISPH context (fluid + static solids; with dynamic solids on a context
 * configured by sph_shard_configure_iisph_bodies, whose additions to the order below are listed there): the step of sph_iisph_step with
 * `io` used the same way, except that io->n_fluid is the GLOBAL fluid count (all ranks).  One step:
 *     plan -> classify + sort -> info -> DX ranges -> ghost alignment -> densities (owned + first ghost layer)
 *     -> non-pressure forces -> predict velocity -> [v*] -> diagonal, source, warm start -> [aux]
 *     -> loop { pressure acceleration -> [acc] -> pressure update (error partial) -> [aux + all-gather of the
 *               partials] -> the loop check on the partials added in rank order }
 *     -> final pressure acceleration -> advect -> fluid wall clamp -> the record exchange
 * ([w] = the 16-byte words w of the outermost owned layer sent to the neighbours' first ghost layer.)  Every rank
 * returns the same iterations, first_batch and avg_err values.  Eager launches with one host wait per batch of sweeps
 * (SPH_SHARD_GRAPH does not apply).  A particle that moves a whole cell layer in x in one step sets
 * SPH_STATUS_SHARD_VELOCITY.  The warm-start pressure travels in the records (misc.y), so migrating particles keep it. */
int sph_shard_iisph_step(SphCtx *ctx, int32_t nsteps, SphIisphStep *io, void *stream);
/* nsteps sharded PCISPH SPHBase.step()s of a context configured by sph_shard_configure_pcisph (fluid + static solids):
 * the step of sph_pcisph_step with `io` used the same way.  One step:
 *     plan -> classify + sort -> info -> DX ranges -> ghost alignment -> densities (owned + first ghost layer)
 *     -> non-pressure forces -> p = 0, a^p = 0, x* = x
 *     -> loop { prediction -> [dfs = {x*, m_V}] -> predicted density + pressure update (error partial) -> [misc.y = p
 *               + all-gather of the partials] -> pressure force -> the loop check on the max of the partials }
 *     -> final pressure force -> advect -> fluid wall clamp -> the record exchange
 * ([w] as for sph_shard_iisph_step.)  The max of the ranks' partials is exact and independent of order, so every rank
 * runs the same sweeps and returns the same iterations, first_batch and max_err values (max_err bit-identical).  Eager
 * launches with one host wait per batch of sweeps (SPH_SHARD_GRAPH does not apply).  A particle that moves a whole
 * cell layer in x in one step sets SPH_STATUS_SHARD_VELOCITY. */
int sph_shard_pcisph_step(SphCtx *ctx, int32_t nsteps, SphPcisphStep *io, void *stream);
/* out2 = {transport groups this context issued from the host, bytes it sent in them}; graph replays of
 * sph_shard_step (SPH_SHARD_GRAPH=1) re-issue the captured groups without counting them */
int sph_shard_transport_stats(SphCtx *ctx, uint64_t *out2);
/* the exchange alone: sends the packed staging, receives behind the live records (SURVEY.md section 8b) */
int sph_halo_exchange(SphCtx *ctx, void *stream);
/* synchronising read of the device-resident step state: out16 = {n_live, owned, x_lo, x_hi, step, own_begin,
 * own_end, sendL_begin, sendL_end, sendR_begin, sendR_end, recv_left, recv_right, n_sorted, status,
 * 0}; out_sent (may be NULL) = halo records sent so far */
int sph_shard_info(SphCtx *ctx, int32_t *out16, uint64_t *out_sent, void *stream);
/* Output of a sharded run: x and v of ONE object gathered on rank 0 (ParticleSystem.dump, particle_system.py:409-418).
 * Collective over the sharded context's ranks, synchronising; call it on every rank at the same point between steps,
 * with the same object_id.  x, v: [capacity, 3] float32 device buffers (the layout of sph_unpack_xv).
 *   - Each rank takes its owned records -- the index range [own_begin, own_end) of the last sort without the ghost
 *     flag, a partition of the particles -- whose object id is object_id, and compacts their x and v on the device
 *     in its sorted order (deterministic, no atomics).
 *   - One transport group: every rank sends {capacity, rows, status word} (16 bytes) to every other rank, so every rank
 *     evaluates the same check: if rank 0's capacity is below the total rows, or any rank's capacity below its own
 *     rows, EVERY rank returns SPH_E_CAPACITY (the message names the capacity) and no rank transfers anything.
 *   - A second group (only if a rank other than 0 holds rows): each rank r > 0 with rows sends them to rank 0, which
 *     receives them behind the rows of ranks 0 .. r - 1; rank 0's own rows are at row 0.
 * On rank 0 *rows_out is the total and x / v hold every rank's rows in rank order; slabs are contiguous x-layer
 * ranges in rank order and the cell flattening is x-major, so that is the global cell order of the last sort.  On
 * the other ranks *rows_out is their own row count and x / v hold their own rows.  *status_out is the OR of every
 * rank's status word (sph_shard_info's), the same on every rank, also when SPH_E_CAPACITY is returned.
 * sph_shard_transport_stats counts the bytes like any other group: this rank sends (world - 1) * 16 bytes of headers,
 * plus, on ranks other than rank 0, 24 bytes (x and v, 3 float32 each) per row it holds.  Launches nothing into
 * sph_shard_step's graphs; works on WCSPH, DFSPH, IISPH, PCISPH and sph_shard_configure_bodies contexts.  Single-GPU contexts are
 * refused (they have sph_unpack_xv); capacity < 0 or a null pointer returns SPH_E_ARG. */
int sph_shard_dump(SphCtx *ctx, int32_t object_id, float *x, float *v, int64_t capacity, int64_t *rows_out,
                   uint32_t *status_out, void *stream);
/* ONE un-graphed sharded step with CUDA events between its stages; ms_out6 = {plan + sort + info, boundary
 * densities, boundary forces (-> staging), interior densities, apply + interior forces (+ waiting for the exchange,
 * if it is not hidden), the exchange alone on the communication stream}; synchronises */
int sph_shard_profile_step(SphCtx *ctx, float *ms_out6, void *stream);
int sph_state_offsets(SphCtx *ctx, uint64_t *out5); /* byte offsets of posm, veld, x0id, misc, acc in the workspace */

/* ---- diagnostics ----------------------------------------------------------------------------- */
int sph_read_status(SphCtx *ctx, uint32_t *status_out, void *stream); /* synchronises `stream` */
int sph_clear_status(SphCtx *ctx, void *stream);
/* neighbour-list statistics of the last density pass: out_dev4 = {max neighbours, particles in the
 * over-full fallback (> 96 neighbours), accepted pairs, fluid particles} */
int sph_neighbor_stats(SphCtx *ctx, int32_t *out_dev4, void *stream);
int64_t sph_particle_count(const SphCtx *ctx);
/* number of kernels launched by this context since creation (graph replays counted per node) */
int64_t sph_launch_count(const SphCtx *ctx);
/* per-kernel timing of ONE un-graphed step with CUDA events on `stream`; synchronises.
 * ms[] receives up to n entries in the order of sph_timer_name(i). Returns entries written. */
int sph_profile_step(SphCtx *ctx, float *ms, int32_t n, void *stream);
const char *sph_timer_name(int32_t i);

#ifdef __cplusplus
}
#endif
#endif /* SPH_B200_H */
