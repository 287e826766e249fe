/*
 * sph_oracle.c -- CPU restatement of the reference WCSPH step (TEST INFRASTRUCTURE ONLY).
 *
 * PARITY PIN: the reference (erizmr/SPH_Taichi @ 4a701fd) ships no tests, golden vectors or
 * fixtures, and the Taichi wheel is not available here.  This file restates the reference's
 * algorithm line by line and is pinned three ways:
 *   (1) tests/test_golden_reference.py -- golden vectors written by the reference's OWN source
 *       files (particle_system.py, sph_base.py, WCSPH.py, DFSPH.py, imported unmodified from
 *       a reference checkout) executed under a pure-Python stand-in for the Taichi runtime
 *       (tests/golden/ti_shim/: serial loops, IEEE float32; tests/golden/make_reference_golden.py).
 *       This pins the algorithm as written in the reference; it is NOT a run of Taichi's
 *       code generator (fast-math, atomics order), which remains unavailable offline;
 *   (2) closed-form known answers (tests/test_oracle.py);
 *   (3) an independent all-pairs numpy restatement (oracle/np_ref.py).
 *
 * Nothing in the product path (sph_taichi_b200/) may import, link or call this file.
 * It is used by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs only.
 *
 * Build: see oracle/Makefile (REAL = float by default; -DORACLE_F64 for the fp64
 * noise-floor variant).  Floating-point contraction is disabled so that the fp32
 * build evaluates exactly the operation sequence written here.
 *
 * Reference files restated (file:line relative to the reference root):
 *   particle_system.py:287-294  pos_to_index / flatten_grid_index
 *   particle_system.py:311-320  update_grid_id
 *   particle_system.py:322-369  counting_sort   (serial semantics = stable sort)
 *   particle_system.py:378-385  for_all_neighbors
 *   sph_base.py:23-68           cubic_kernel / cubic_kernel_derivative
 *   sph_base.py:91-113          compute_static/moving_boundary_volume
 *   sph_base.py:118-123,149-179 simulate_collisions / enforce_boundary_3D
 *   sph_base.py:182-222,247-260 compute_com / solve_constraints / solve_rigid_body
 *   sph_base.py:263-271         step
 *   WCSPH.py:19-43              compute_densities
 *   WCSPH.py:46-85              compute_pressure_forces
 *   WCSPH.py:88-140             compute_non_pressure_forces
 *   WCSPH.py:143-156            advect / substep
 *   DFSPH.py:116-227,278-311,354-408  DFSPH factor, density change / adv, error, Jacobi iteration kernels,
 *                                predict_velocity, advect (simulationMethod 4; host loops live in sph_oracle.py)
 *
 * Conscious, tested deviations from the literal reference (SURVEY.md section 8 Q-list):
 *   Q3  neighbour cells with any axis index out of [0, grid_num) are skipped (the
 *       reference reads aliased / out-of-bounds cells there; the aliased cells can never
 *       pass the r < h test for grids >= 3 cells per axis).
 *   Q7  the counting sort is stable (serial semantics of the reference loop); reaction
 *       forces on dynamic rigid particles are summed in ascending fluid index (the
 *       reference uses unordered float atomics).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double REAL;
#define R_SQRT sqrt
#define R_POW pow
#define R_FABS fabs
#else
typedef float REAL;
#define R_SQRT sqrtf
#define R_POW powf
#define R_FABS fabsf
#endif

typedef struct {
    int32_t n;             /* particle count (== particle_max_num, no emitter) */
    int32_t grid_num[3];   /* ceil(domain_size / h) */
    REAL h;                /* support radius = grid size = padding */
    REAL diameter;         /* particle diameter */
    REAL m_V0;             /* 0.8 d^3 */
    REAL density0;
    REAL stiffness;
    REAL exponent;
    REAL viscosity;        /* 0.01 */
    REAL surface_tension;  /* 0.01 */
    REAL dt;
    REAL g[3];
    REAL domain_size[3];
    REAL k_w;              /* 8 / (pi h^3), folded in double on the host like the reference */
    REAL k_dw;             /* 6 * k_w */
    REAL visc_eps;         /* 0.01 h^2 */
} OracleParams;

typedef struct {
    int32_t *object_id;
    REAL *x, *x_0, *v, *acceleration; /* [n][3] */
    REAL *m_V, *m, *density, *pressure;
    int32_t *material, *is_dynamic;
    int32_t *color;                   /* [n][3] */
    int32_t *grid_ids;                /* [n] */
    int32_t *grid_particles_num;      /* [C]; after neighbour build: inclusive prefix sum */
    REAL *dfsph_factor, *density_adv; /* DFSPH only (particle_system.py:115-117); may be NULL */
} OracleState;

#define MAT_SOLID 0
#define MAT_FLUID 1

int oracle_real_bytes(void) { return (int)sizeof(REAL); }

/* ---- particle_system.py:287-294 -------------------------------------------------- */
static inline void pos_to_index(const OracleParams *P, const REAL *pos, int32_t idx[3]) {
    for (int a = 0; a < 3; ++a) idx[a] = (int32_t)(pos[a] / P->h); /* trunc toward zero */
}
static inline int32_t flatten(const OracleParams *P, const int32_t idx[3]) {
    return idx[0] * P->grid_num[1] * P->grid_num[2] + idx[1] * P->grid_num[2] + idx[2];
}
static inline int64_t cell_count(const OracleParams *P) {
    return (int64_t)P->grid_num[0] * P->grid_num[1] * P->grid_num[2];
}

/* ---- sph_base.py:23-44 ------------------------------------------------------------ */
static inline REAL cubic_kernel(const OracleParams *P, REAL r_norm) {
    REAL res = (REAL)0.0;
    REAL q = r_norm / P->h;
    if (q <= (REAL)1.0) {
        if (q <= (REAL)0.5) {
            REAL q2 = q * q;
            REAL q3 = q2 * q;
            res = P->k_w * ((REAL)6.0 * q3 - (REAL)6.0 * q2 + (REAL)1.0);
        } else {
            res = (P->k_w * (REAL)2.0) * R_POW((REAL)1.0 - q, (REAL)3.0);
        }
    }
    return res;
}

/* ---- sph_base.py:46-68 ------------------------------------------------------------ */
static inline void cubic_kernel_derivative(const OracleParams *P, const REAL r[3], REAL out[3]) {
    REAL r_norm = R_SQRT(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    REAL q = r_norm / P->h;
    out[0] = out[1] = out[2] = (REAL)0.0;
    if (r_norm > (REAL)1e-5 && q <= (REAL)1.0) {
        REAL den = r_norm * P->h;
        REAL s;
        if (q <= (REAL)0.5) {
            s = P->k_dw * q * ((REAL)3.0 * q - (REAL)2.0);
        } else {
            REAL f = (REAL)1.0 - q;
            s = P->k_dw * (-f * f);
        }
        for (int a = 0; a < 3; ++a) out[a] = s * (r[a] / den);
    }
}

static inline REAL norm3(const REAL r[3]) { return R_SQRT(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]); }

/* ---- particle_system.py:311-375 --------------------------------------------------- */
static void permute_real(REAL *a, const int32_t *dst, int32_t n, int w, void *tmp) {
    REAL *t = (REAL *)tmp;
#pragma omp parallel for schedule(static)
    for (int32_t i = 0; i < n; ++i)
        for (int c = 0; c < w; ++c) t[(size_t)dst[i] * w + c] = a[(size_t)i * w + c];
    memcpy(a, t, sizeof(REAL) * (size_t)n * w);
}
static void permute_i32(int32_t *a, const int32_t *dst, int32_t n, int w, void *tmp) {
    int32_t *t = (int32_t *)tmp;
#pragma omp parallel for schedule(static)
    for (int32_t i = 0; i < n; ++i)
        for (int c = 0; c < w; ++c) t[(size_t)dst[i] * w + c] = a[(size_t)i * w + c];
    memcpy(a, t, sizeof(int32_t) * (size_t)n * w);
}

/* update_grid_id + inclusive prefix sum + counting sort.  Returns 0, or -1 when a particle
 * hashes outside the grid (the reference would write out of bounds). */
int oracle_neighbor_build(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
    const int64_t C = cell_count(P);
    int32_t *cnt = S->grid_particles_num;
    memset(cnt, 0, sizeof(int32_t) * (size_t)C);
    int bad = 0;
#pragma omp parallel for schedule(static) reduction(| : bad)
    for (int32_t i = 0; i < n; ++i) {
        int32_t idx[3];
        pos_to_index(P, S->x + 3 * (size_t)i, idx);
        int32_t c = flatten(P, idx);
        if (c < 0 || c >= C) { bad |= 1; c = 0; }
        S->grid_ids[i] = c;
    }
    if (bad) return -1;
    for (int32_t i = 0; i < n; ++i) cnt[S->grid_ids[i]] += 1; /* serial histogram: deterministic */
    /* PrefixSumExecutor.run: in-place inclusive scan (particle_system.py:374) */
    for (int64_t c = 1; c < C; ++c) cnt[c] += cnt[c - 1];
    /* stable counting sort (serial semantics of particle_system.py:325-330) */
    int32_t *fill = (int32_t *)calloc((size_t)C, sizeof(int32_t));
    int32_t *dst = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    void *tmp = malloc(sizeof(double) * 3 * (size_t)(n > 0 ? n : 1));
    if (!fill || !dst || !tmp) { free(fill); free(dst); free(tmp); return -2; }
    for (int32_t i = 0; i < n; ++i) {
        int32_t c = S->grid_ids[i];
        int32_t base = (c - 1 >= 0) ? cnt[c - 1] : 0;
        dst[i] = base + fill[c]++;
    }
    permute_i32(S->grid_ids, dst, n, 1, tmp);
    permute_i32(S->object_id, dst, n, 1, tmp);
    permute_real(S->x_0, dst, n, 3, tmp);
    permute_real(S->x, dst, n, 3, tmp);
    permute_real(S->v, dst, n, 3, tmp);
    permute_real(S->acceleration, dst, n, 3, tmp);
    permute_real(S->m_V, dst, n, 1, tmp);
    permute_real(S->m, dst, n, 1, tmp);
    permute_real(S->density, dst, n, 1, tmp);
    permute_real(S->pressure, dst, n, 1, tmp);
    permute_i32(S->material, dst, n, 1, tmp);
    permute_i32(S->color, dst, n, 3, tmp);
    permute_i32(S->is_dynamic, dst, n, 1, tmp);
    if (S->dfsph_factor) permute_real(S->dfsph_factor, dst, n, 1, tmp); /* particle_system.py:348-350 */
    if (S->density_adv) permute_real(S->density_adv, dst, n, 1, tmp);
    free(fill); free(dst); free(tmp);
    return 0;
}

/* ---- particle_system.py:378-385: neighbour iteration as a macro-style helper -------- */
#define FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)                                                   \
    {                                                                                             \
        int32_t _cc[3];                                                                           \
        pos_to_index((P), (S)->x + 3 * (size_t)(p_i), _cc);                                       \
        for (int _ox = -1; _ox <= 1; ++_ox)                                                       \
            for (int _oy = -1; _oy <= 1; ++_oy)                                                   \
                for (int _oz = -1; _oz <= 1; ++_oz) {                                             \
                    int32_t _nc[3] = {_cc[0] + _ox, _cc[1] + _oy, _cc[2] + _oz};                  \
                    if (_nc[0] < 0 || _nc[0] >= (P)->grid_num[0] || _nc[1] < 0 ||                 \
                        _nc[1] >= (P)->grid_num[1] || _nc[2] < 0 || _nc[2] >= (P)->grid_num[2])   \
                        continue; /* Q3 fence */                                                  \
                    int32_t _g = flatten((P), _nc);                                               \
                    int32_t _lo = (S)->grid_particles_num[_g - 1 > 0 ? _g - 1 : 0];               \
                    int32_t _hi = (S)->grid_particles_num[_g];                                    \
                    for (int32_t p_j = _lo; p_j < _hi; ++p_j) {                                   \
                        if ((p_i) == p_j) continue;                                               \
                        REAL _r[3] = {(S)->x[3 * (size_t)(p_i)] - (S)->x[3 * (size_t)p_j],        \
                                      (S)->x[3 * (size_t)(p_i) + 1] - (S)->x[3 * (size_t)p_j + 1],\
                                      (S)->x[3 * (size_t)(p_i) + 2] - (S)->x[3 * (size_t)p_j + 2]};\
                        if (!(norm3(_r) < (P)->h)) continue;

#define FOR_ALL_NEIGHBORS_END                                                                     \
                    }                                                                             \
                }                                                                                 \
    }

static inline int is_static_rigid(const OracleState *S, int32_t p) {
    return S->material[p] == MAT_SOLID && !S->is_dynamic[p];
}
static inline int is_dynamic_rigid(const OracleState *S, int32_t p) {
    return S->material[p] == MAT_SOLID && S->is_dynamic[p];
}

/* ---- sph_base.py:91-113: moving = 0 -> static bodies, 1 -> dynamic bodies ----------- */
void oracle_boundary_volume(const OracleParams *P, OracleState *S, int moving) {
    const int32_t n = P->n;
    REAL *out = (REAL *)malloc(sizeof(REAL) * (size_t)(n > 0 ? n : 1));
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        int sel = moving ? is_dynamic_rigid(S, p_i) : is_static_rigid(S, p_i);
        out[p_i] = S->m_V[p_i];
        if (!sel) continue;
        REAL delta = cubic_kernel(P, (REAL)0.0);
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            if (S->material[p_j] == MAT_SOLID) delta += cubic_kernel(P, norm3(_r));
        FOR_ALL_NEIGHBORS_END
        out[p_i] = (REAL)1.0 / delta * (REAL)3.0;
    }
    /* m_V is only read for solid neighbours' *positions* above, so in-place == two-phase */
    memcpy(S->m_V, out, sizeof(REAL) * (size_t)n);
    free(out);
}

/* ---- WCSPH.py:19-43 ---------------------------------------------------------------- */
void oracle_compute_densities(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        if (S->material[p_i] != MAT_FLUID) continue;
        REAL rho = S->m_V[p_i] * cubic_kernel(P, (REAL)0.0);
        REAL den = (REAL)0.0;
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            /* fluid and solid neighbours use the same expression (WCSPH.py:22-30) */
            den += S->m_V[p_j] * cubic_kernel(P, norm3(_r));
        FOR_ALL_NEIGHBORS_END
        rho += den;
        rho *= P->density0;
        S->density[p_i] = rho;
    }
}

/* ---- WCSPH.py:88-140 --------------------------------------------------------------- */
void oracle_compute_non_pressure_forces(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
    const REAL d_visc = (REAL)(2.0 * (3 + 2)) * P->viscosity; /* d * viscosity folded on host */
    const REAL diameter2 = P->diameter * P->diameter;
    const REAL w_diam = cubic_kernel(P, P->diameter); /* ||(d,0,0)|| = d */
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        REAL *a = S->acceleration + 3 * (size_t)p_i;
        if (is_static_rigid(S, p_i)) { a[0] = a[1] = a[2] = (REAL)0.0; continue; }
        REAL dv[3] = {P->g[0], P->g[1], P->g[2]};
        if (S->material[p_i] == MAT_FLUID) {
            FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
                REAL r2 = _r[0] * _r[0] + _r[1] * _r[1] + _r[2] * _r[2];
                if (S->material[p_j] == MAT_FLUID) {
                    /* surface tension (cohesion), WCSPH.py:93-103 */
                    REAL w = (r2 > diameter2) ? cubic_kernel(P, norm3(_r)) : w_diam;
                    REAL c = P->surface_tension / S->m[p_i] * S->m[p_j];
                    for (int k = 0; k < 3; ++k) dv[k] -= c * _r[k] * w;
                    /* viscosity, WCSPH.py:106-116 (rho_j is the UNCLAMPED density, Q4) */
                    const REAL *vi = S->v + 3 * (size_t)p_i, *vj = S->v + 3 * (size_t)p_j;
                    REAL v_xy = (vi[0] - vj[0]) * _r[0] + (vi[1] - vj[1]) * _r[1] + (vi[2] - vj[2]) * _r[2];
                    REAL rn = norm3(_r);
                    REAL s = d_visc * (S->m[p_j] / S->density[p_j]) * v_xy / (rn * rn + P->visc_eps);
                    REAL gw[3];
                    cubic_kernel_derivative(P, _r, gw);
                    for (int k = 0; k < 3; ++k) dv[k] += s * gw[k];
                }
                /* solid neighbours: boundary_viscosity == 0.0 -> exact zeros (WCSPH.py:117-125) */
                (void)r2;
            FOR_ALL_NEIGHBORS_END
        }
        a[0] = dv[0]; a[1] = dv[1]; a[2] = dv[2];
    }
}

/* ---- WCSPH.py:46-85 ---------------------------------------------------------------- */
static inline void pressure_pair_solid(const OracleParams *P, const OracleState *S, int32_t p_i, int32_t p_j,
                                       const REAL r[3], REAL f_p[3]) {
    REAL dpi = S->pressure[p_i] / (S->density[p_i] * S->density[p_i]);
    REAL dpj = S->pressure[p_i] / (P->density0 * P->density0);
    REAL gw[3];
    cubic_kernel_derivative(P, r, gw);
    REAL c = -P->density0 * S->m_V[p_j] * (dpi + dpj);
    for (int k = 0; k < 3; ++k) f_p[k] = c * gw[k];
}

void oracle_compute_pressure_forces(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
#pragma omp parallel for schedule(static)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        if (S->material[p_i] != MAT_FLUID) continue;
        REAL rho = S->density[p_i];
        if (!(rho > P->density0)) rho = P->density0; /* ti.max */
        S->density[p_i] = rho;
        S->pressure[p_i] = P->stiffness * (R_POW(rho / P->density0, P->exponent) - (REAL)1.0);
    }
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        REAL *a = S->acceleration + 3 * (size_t)p_i;
        if (is_static_rigid(S, p_i)) { a[0] = a[1] = a[2] = (REAL)0.0; continue; }
        if (is_dynamic_rigid(S, p_i)) {
            /* gather form of the reference's atomic scatter (WCSPH.py:66-68): every fluid
             * neighbour p_f of this rigid particle contributes -f_p(p_f, p_i) * rho0 / rho_i */
            REAL acc[3] = {0, 0, 0};
            FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
                if (S->material[p_j] == MAT_FLUID) {
                    REAL rr[3] = {-_r[0], -_r[1], -_r[2]}; /* x_f - x_rigid */
                    REAL f_p[3];
                    pressure_pair_solid(P, S, p_j, p_i, rr, f_p);
                    for (int k = 0; k < 3; ++k) acc[k] += -f_p[k] * P->density0 / S->density[p_i];
                }
            FOR_ALL_NEIGHBORS_END
            for (int k = 0; k < 3; ++k) a[k] += acc[k];
            continue;
        }
        REAL dv[3] = {0, 0, 0};
        REAL dpi = S->pressure[p_i] / (S->density[p_i] * S->density[p_i]);
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            if (S->material[p_j] == MAT_FLUID) {
                REAL density_j = S->density[p_j] * P->density0 / P->density0; /* WCSPH.py:53 */
                REAL dpj = S->pressure[p_j] / (density_j * density_j);
                REAL gw[3];
                cubic_kernel_derivative(P, _r, gw);
                REAL c = -P->density0 * S->m_V[p_j] * (dpi + dpj);
                for (int k = 0; k < 3; ++k) dv[k] += c * gw[k];
            } else {
                REAL f_p[3];
                pressure_pair_solid(P, S, p_i, p_j, _r, f_p);
                for (int k = 0; k < 3; ++k) dv[k] += f_p[k];
            }
        FOR_ALL_NEIGHBORS_END
        for (int k = 0; k < 3; ++k) a[k] += dv[k];
    }
}

/* ---- WCSPH.py:143-149 -------------------------------------------------------------- */
void oracle_advect(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
#pragma omp parallel for schedule(static)
    for (int32_t p = 0; p < n; ++p) {
        if (!S->is_dynamic[p]) continue;
        for (int k = 0; k < 3; ++k) {
            S->v[3 * (size_t)p + k] += P->dt * S->acceleration[3 * (size_t)p + k];
            S->x[3 * (size_t)p + k] += P->dt * S->v[3 * (size_t)p + k];
        }
    }
}

/* ---- sph_base.py:118-123,149-179 ---------------------------------------------------- */
void oracle_enforce_boundary_3D(const OracleParams *P, OracleState *S, int particle_type) {
    const int32_t n = P->n;
    const REAL pad = P->h;
#pragma omp parallel for schedule(static)
    for (int32_t p = 0; p < n; ++p) {
        if (!(S->material[p] == particle_type && S->is_dynamic[p])) continue;
        REAL *x = S->x + 3 * (size_t)p, *v = S->v + 3 * (size_t)p;
        REAL pos[3] = {x[0], x[1], x[2]};
        REAL nrm[3] = {0, 0, 0};
        for (int k = 0; k < 3; ++k) {
            REAL hi = P->domain_size[k] - pad; /* folded on the host in the reference */
            if (pos[k] > hi) { nrm[k] += (REAL)1.0; x[k] = hi; }
            if (pos[k] <= pad) { nrm[k] += (REAL)-1.0; x[k] = pad; }
        }
        REAL len = norm3(nrm);
        if (len > (REAL)1e-6) {
            REAL u[3] = {nrm[0] / len, nrm[1] / len, nrm[2] / len};
            REAL vd = v[0] * u[0] + v[1] * u[1] + v[2] * u[2];
            REAL f = ((REAL)1.0 + (REAL)0.5) * vd;
            for (int k = 0; k < 3; ++k) v[k] -= f * u[k];
        }
    }
}

/* ---- sph_base.py:182-192 ------------------------------------------------------------ */
void oracle_compute_com(const OracleParams *P, const OracleState *S, int object_id, REAL cm[3]) {
    REAL sum_m = (REAL)0.0;
    cm[0] = cm[1] = cm[2] = (REAL)0.0;
    for (int32_t p = 0; p < P->n; ++p) {
        if (is_dynamic_rigid(S, p) && S->object_id[p] == object_id) {
            REAL mass = P->m_V0 * S->density[p];
            for (int k = 0; k < 3; ++k) cm[k] += mass * S->x[3 * (size_t)p + k];
            sum_m += mass;
        }
    }
    for (int k = 0; k < 3; ++k) cm[k] /= sum_m; /* 0/0 = NaN for static bodies (Q8) */
}

/* Rotation factor of the polar decomposition A = R S (what ti.polar_decompose returns for
 * R; Taichi derives it from an SVD, R = U V^T).  Here: scaled Newton iteration on
 * X <- (X + X^-T) / 2 in double precision; for non-singular A the factor is unique. */
static void polar_rotation(const double A[9], double R[9]) {
    double X[9];
    memcpy(X, A, sizeof(X));
    for (int it = 0; it < 100; ++it) {
        double c[9]; /* cofactor matrix: X^-T = cof / det */
        c[0] = X[4] * X[8] - X[5] * X[7]; c[1] = X[5] * X[6] - X[3] * X[8]; c[2] = X[3] * X[7] - X[4] * X[6];
        c[3] = X[2] * X[7] - X[1] * X[8]; c[4] = X[0] * X[8] - X[2] * X[6]; c[5] = X[1] * X[6] - X[0] * X[7];
        c[6] = X[1] * X[5] - X[2] * X[4]; c[7] = X[2] * X[3] - X[0] * X[5]; c[8] = X[0] * X[4] - X[1] * X[3];
        double det = X[0] * c[0] + X[1] * c[1] + X[2] * c[2];
        if (fabs(det) < 1e-300) break;
        double nx = 0, ni = 0;
        for (int i = 0; i < 9; ++i) { nx += X[i] * X[i]; ni += (c[i] / det) * (c[i] / det); }
        double gamma = sqrt(sqrt(ni / nx)); /* Frobenius-norm scaling */
        double diff = 0;
        for (int i = 0; i < 9; ++i) {
            double y = 0.5 * (gamma * X[i] + (c[i] / det) / gamma);
            diff += (y - X[i]) * (y - X[i]);
            X[i] = y;
        }
        if (diff < 1e-30) break;
    }
    memcpy(R, X, sizeof(X));
    /* The iteration yields the orthogonal polar factor Q with det Q = sign(det A).  ti.polar_decompose builds R from
     * an SVD with proper rotations U, V (the sign goes to the smallest singular value): for det A < 0 that is
     * R = Q (I - 2 v v^T), v = eigenvector of S = Q^T A with the smallest eigenvalue (cyclic Jacobi below). */
    double detA = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    if (detA < 0.0) {
        double S[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) S[3 * r + c] = X[r] * A[c] + X[3 + r] * A[3 + c] + X[6 + r] * A[6 + c];
        for (int r = 0; r < 3; ++r)
            for (int c = r + 1; c < 3; ++c) S[3 * r + c] = S[3 * c + r] = 0.5 * (S[3 * r + c] + S[3 * c + r]);
        for (int sweep = 0; sweep < 12; ++sweep)
            for (int p = 0; p < 2; ++p)
                for (int q = p + 1; q < 3; ++q) {
                    double apq = S[3 * p + q];
                    if (fabs(apq) < 1e-300) continue;
                    double th = 0.5 * (S[3 * q + q] - S[3 * p + p]) / apq;
                    double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                    double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
                    for (int k = 0; k < 3; ++k) {
                        double skp = S[3 * k + p], skq = S[3 * k + q];
                        S[3 * k + p] = cs * skp - sn * skq; S[3 * k + q] = sn * skp + cs * skq;
                    }
                    for (int k = 0; k < 3; ++k) {
                        double spk = S[3 * p + k], sqk = S[3 * q + k];
                        S[3 * p + k] = cs * spk - sn * sqk; S[3 * q + k] = sn * spk + cs * sqk;
                        double vkp = V[3 * k + p], vkq = V[3 * k + q];
                        V[3 * k + p] = cs * vkp - sn * vkq; V[3 * k + q] = sn * vkp + cs * vkq;
                    }
                }
        int m = 0;
        if (S[4] < S[3 * m + m]) m = 1;
        if (S[8] < S[3 * m + m]) m = 2;
        double v[3] = {V[m], V[3 + m], V[6 + m]};
        for (int r = 0; r < 3; ++r) {
            double qv = X[3 * r] * v[0] + X[3 * r + 1] * v[1] + X[3 * r + 2] * v[2];
            for (int c = 0; c < 3; ++c) R[3 * r + c] = X[3 * r + c] - 2.0 * qv * v[c];
        }
    }
}

/* ---- sph_base.py:200-222: returns R (row-major) ------------------------------------- */
void oracle_solve_constraints(const OracleParams *P, OracleState *S, int object_id, const REAL rest_cm[3],
                              REAL R_out[9]) {
    REAL cm[3];
    oracle_compute_com(P, S, object_id, cm);
    REAL A[9] = {0};
    for (int32_t p = 0; p < P->n; ++p) {
        if (is_dynamic_rigid(S, p) && S->object_id[p] == object_id) {
            REAL q[3], pp[3];
            for (int k = 0; k < 3; ++k) {
                q[k] = S->x_0[3 * (size_t)p + k] - rest_cm[k];
                pp[k] = S->x[3 * (size_t)p + k] - cm[k];
            }
            REAL w = P->m_V0 * S->density[p];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) A[3 * r + c] += w * pp[r] * q[c];
        }
    }
    double Ad[9], Rd[9];
    for (int i = 0; i < 9; ++i) Ad[i] = (double)A[i];
    polar_rotation(Ad, Rd);
    REAL R[9];
    int all_small = 1;
    for (int i = 0; i < 9; ++i) { R[i] = (REAL)Rd[i]; if (!(R_FABS(R[i]) < (REAL)1e-6)) all_small = 0; }
    if (all_small) { memset(R, 0, sizeof(R)); R[0] = R[4] = R[8] = (REAL)1.0; }
    for (int32_t p = 0; p < P->n; ++p) {
        if (is_dynamic_rigid(S, p) && S->object_id[p] == object_id) {
            REAL q[3];
            for (int k = 0; k < 3; ++k) q[k] = S->x_0[3 * (size_t)p + k] - rest_cm[k];
            for (int r = 0; r < 3; ++r) {
                REAL goal = cm[r] + (R[3 * r] * q[0] + R[3 * r + 1] * q[1] + R[3 * r + 2] * q[2]);
                REAL corr = (goal - S->x[3 * (size_t)p + r]) * (REAL)1.0;
                S->x[3 * (size_t)p + r] += corr;
            }
        }
    }
    memcpy(R_out, R, sizeof(R));
}

/* ---- sph_base.py:263-271 + WCSPH.py:152-156: one full step --------------------------- */
/* dyn_ids / rest_cms: the dynamic rigid bodies in iteration order (set of object ids) */
int oracle_step(const OracleParams *P, OracleState *S, int n_dyn, const int32_t *dyn_ids, const REAL *rest_cms) {
    int rc = oracle_neighbor_build(P, S);
    if (rc) return rc;
    oracle_boundary_volume(P, S, 1);
    oracle_compute_densities(P, S);
    oracle_compute_non_pressure_forces(P, S);
    oracle_compute_pressure_forces(P, S);
    oracle_advect(P, S);
    for (int b = 0; b < n_dyn; ++b) {
        REAL R[9];
        oracle_solve_constraints(P, S, dyn_ids[b], rest_cms + 3 * b, R);
        oracle_enforce_boundary_3D(P, S, MAT_SOLID);
    }
    oracle_enforce_boundary_3D(P, S, MAT_FLUID);
    return 0;
}


/* ==================================================================================== */
/* DFSPH (reference DFSPH.py, simulationMethod 4).  compute_densities and                */
/* compute_non_pressure_forces are the WCSPH functions above (DFSPH.py:24-47, 50-101 are  */
/* the same expressions; the only difference, the reaction of the boundary viscosity, is  */
/* multiplied by boundary_viscosity = 0.0).                                               */
/* ==================================================================================== */

/* DFSPH.py:114-154 */
void oracle_dfsph_compute_factor(const OracleParams *P, OracleState *S) {
    const int32_t n = P->n;
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        if (S->material[p_i] != MAT_FLUID) continue;
        REAL ret[4] = {0, 0, 0, 0};
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            REAL gw[3];
            cubic_kernel_derivative(P, _r, gw);
            REAL g[3] = {-S->m_V[p_j] * gw[0], -S->m_V[p_j] * gw[1], -S->m_V[p_j] * gw[2]};
            if (S->material[p_j] == MAT_FLUID) ret[3] += g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
            for (int k = 0; k < 3; ++k) ret[k] -= g[k];
        FOR_ALL_NEIGHBORS_END
        REAL sum_grad_p_k = ret[3];
        sum_grad_p_k += ret[0] * ret[0] + ret[1] * ret[1] + ret[2] * ret[2];
        S->dfsph_factor[p_i] = (sum_grad_p_k > (REAL)1e-6) ? (REAL)-1.0 / sum_grad_p_k : (REAL)0.0;
    }
}

/* DFSPH.py:157-196 (mode 0: compute_density_change) and :198-219 (mode 1: compute_density_adv) */
void oracle_dfsph_density_change(const OracleParams *P, OracleState *S, int mode) {
    const int32_t n = P->n;
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        if (S->material[p_i] != MAT_FLUID) continue;
        REAL acc = (REAL)0.0;
        int32_t nn = 0;
        const REAL *vi = S->v + 3 * (size_t)p_i;
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            REAL gw[3];
            cubic_kernel_derivative(P, _r, gw);
            const REAL *vj = S->v + 3 * (size_t)p_j;
            acc += S->m_V[p_j] * ((vi[0] - vj[0]) * gw[0] + (vi[1] - vj[1]) * gw[1] + (vi[2] - vj[2]) * gw[2]);
            nn += 1;
        FOR_ALL_NEIGHBORS_END
        if (mode == 0) {
            REAL da = acc > (REAL)0.0 ? acc : (REAL)0.0; /* only correct positive divergence */
            if (nn < 20) da = (REAL)0.0;                 /* particle deficiency (3-D) */
            S->density_adv[p_i] = da;
        } else {
            REAL da = S->density[p_i] / P->density0 + P->dt * acc;
            S->density_adv[p_i] = da > (REAL)1.0 ? da : (REAL)1.0;
        }
    }
}

/* DFSPH.py:221-227: serial sum in particle order (the reference reduces with atomics) */
double oracle_dfsph_density_error(const OracleParams *P, const OracleState *S, double offset) {
    REAL err = (REAL)0.0;
    for (int32_t i = 0; i < P->n; ++i)
        if (S->material[i] == MAT_FLUID) err += P->density0 * S->density_adv[i] - (REAL)offset;
    return (double)err;
}

/* DFSPH.py:229-233 on dfsph_factor */
void oracle_dfsph_multiply_factor(const OracleParams *P, OracleState *S, double time_step) {
    for (int32_t i = 0; i < P->n; ++i)
        if (S->material[i] == MAT_FLUID) S->dfsph_factor[i] *= (REAL)time_step;
}

/* DFSPH.py:278-311 (mode 0: divergence_solver_iteration_kernel) and :354-389 (mode 1:
 * pressure_solve_iteration_kernel).  Reactions on dynamic rigid particles: mode 0 adds them to an
 * acceleration that compute_non_pressure_forces overwrites before anybody reads it (DFSPH.py:402),
 * so they are dropped here; mode 1 accumulates them in gather form (deterministic order). */
void oracle_dfsph_iteration(const OracleParams *P, OracleState *S, int mode) {
    const int32_t n = P->n;
    const REAL eps = (REAL)1e-5;
    const REAL boff = mode == 0 ? (REAL)0.0 : (REAL)1.0;
    REAL *vnew = (REAL *)malloc(sizeof(REAL) * 3 * (size_t)(n > 0 ? n : 1));
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t p_i = 0; p_i < n; ++p_i) {
        for (int k = 0; k < 3; ++k) vnew[3 * (size_t)p_i + k] = S->v[3 * (size_t)p_i + k];
        if (S->material[p_i] != MAT_FLUID) continue;
        REAL k_i = (S->density_adv[p_i] - boff) * S->dfsph_factor[p_i];
        REAL dv[3] = {0, 0, 0};
        REAL *vi = vnew + 3 * (size_t)p_i;
        FOR_ALL_NEIGHBORS_BEGIN(P, S, p_i, p_j)
            if (S->material[p_j] == MAT_FLUID) {
                REAL k_j = (S->density_adv[p_j] - boff) * S->dfsph_factor[p_j];
                REAL k_sum = k_i + P->density0 / P->density0 * k_j;
                if (R_FABS(k_sum) > eps) {
                    REAL gw[3];
                    cubic_kernel_derivative(P, _r, gw);
                    for (int k = 0; k < 3; ++k) {
                        REAL gp = -S->m_V[p_j] * gw[k];
                        if (mode == 0) dv[k] -= P->dt * k_sum * gp;
                        else vi[k] -= P->dt * k_sum * gp;
                    }
                }
            } else if (R_FABS(k_i) > eps) {
                REAL gw[3];
                cubic_kernel_derivative(P, _r, gw);
                for (int k = 0; k < 3; ++k) {
                    REAL gp = -S->m_V[p_j] * gw[k];
                    REAL vel_change = -P->dt * (REAL)1.0 * k_i * gp;
                    if (mode == 0) dv[k] += vel_change;
                    else vi[k] += vel_change;
                }
            }
        FOR_ALL_NEIGHBORS_END
        if (mode == 0) for (int k = 0; k < 3; ++k) vi[k] += dv[k];
    }
    if (mode == 1) { /* reactions, DFSPH.py:388-389 */
#pragma omp parallel for schedule(dynamic, 256)
        for (int32_t p_j = 0; p_j < n; ++p_j) {
            if (!is_dynamic_rigid(S, p_j)) continue;
            REAL acc[3] = {0, 0, 0};
            FOR_ALL_NEIGHBORS_BEGIN(P, S, p_j, p_f)
                if (S->material[p_f] == MAT_FLUID) {
                    REAL k_f = (S->density_adv[p_f] - boff) * S->dfsph_factor[p_f];
                    if (R_FABS(k_f) > eps) {
                        REAL rr[3] = {-_r[0], -_r[1], -_r[2]}; /* x_f - x_rigid */
                        REAL gw[3];
                        cubic_kernel_derivative(P, rr, gw);
                        for (int k = 0; k < 3; ++k) {
                            REAL gp = -S->m_V[p_j] * gw[k];
                            REAL vel_change = -P->dt * (REAL)1.0 * k_f * gp;
                            acc[k] += -vel_change * (REAL)1.0 / P->dt * S->density[p_f] / S->density[p_j];
                        }
                    }
                }
            FOR_ALL_NEIGHBORS_END
            for (int k = 0; k < 3; ++k) S->acceleration[3 * (size_t)p_j + k] += acc[k];
        }
    }
    memcpy(S->v, vnew, sizeof(REAL) * 3 * (size_t)n);
    free(vnew);
}

/* DFSPH.py:392-397 */
void oracle_dfsph_predict_velocity(const OracleParams *P, OracleState *S) {
    for (int32_t p = 0; p < P->n; ++p)
        if (S->is_dynamic[p] && S->material[p] == MAT_FLUID)
            for (int k = 0; k < 3; ++k) S->v[3 * (size_t)p + k] += P->dt * S->acceleration[3 * (size_t)p + k];
}

/* DFSPH.py:104-111 */
void oracle_dfsph_advect(const OracleParams *P, OracleState *S) {
    for (int32_t p = 0; p < P->n; ++p) {
        if (!S->is_dynamic[p]) continue;
        for (int k = 0; k < 3; ++k) {
            if (is_dynamic_rigid(S, p)) S->v[3 * (size_t)p + k] += P->dt * S->acceleration[3 * (size_t)p + k];
            S->x[3 * (size_t)p + k] += P->dt * S->v[3 * (size_t)p + k];
        }
    }
}
