// sph_b200.cu -- host side of libsph_b200.so: context, workspace carving, launch sequences,
// CUDA-graph step replay, and the extern "C" ABI declared in include/sph_b200.h.
#include <cuda_runtime.h>
#ifndef SPH_EMU
#include <dlfcn.h>
#endif

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "sph_iisph.cuh"
#include "sph_pcisph.cuh"

namespace {

std::string g_create_error;

// Contexts configured by sph_shard_configure hold static solids only.  The solid-id slot map of a rank is not reset or validated under
// migration (a trash-bucket record may share its id with a live one, a solid on another rank leaves its slot stale),
// so every entry point that walks it -- boundary volumes, advect-solids, the rigid-body calls -- is refused there.
const char *const kShardStaticOnly =
    "x-slab sharding supports static solids only: dynamic solids (shape-matched bodies, advected rigid blocks) and "
    "the rigid-body and boundary-volume calls that walk solid ids are single-GPU in WCSPH and DFSPH";
// sph_shard_configure_bodies (opt-in, WCSPH): the step re-validates the slot map and solves the bodies across ranks
const char *const kShardBodiesWcsph =
    "x-slab sharding of dynamic solids is WCSPH only: the DFSPH pressure sweeps scatter the reactions onto the bodies "
    "in every sweep, which would need a reaction exchange per sweep";
const char *const kIisphContext =
    "this context is in IISPH mode (sph_set_iisph): it steps with sph_iisph_op / sph_iisph_solve / sph_iisph_step";
// sharded IISPH (sph_shard_iisph_step) runs fluid and static solids; the single-GPU IISPH calls launch over the
// capacity of a sharded context and would step its ghost and trash records too
const char *const kIisphSharded = "this IISPH context is sharded: step it with sph_shard_iisph_step";
const char *const kIisphShardStep =
    "this context is in IISPH mode (sph_set_iisph): a sharded IISPH context steps with sph_shard_iisph_step";
const char *const kIisphAfterConfigure = "call sph_set_iisph(1) before sph_shard_configure, not on a sharded context";
const char *const kShardBodiesIisph =
    "x-slab sharding of dynamic solids is WCSPH only: dynamic solids in IISPH are single-GPU unless requested: "
    "sph_shard_configure_iisph_bodies";
const char *const kShardIisphBodiesContext =
    "sph_shard_configure_iisph_bodies shards the dynamic solids of an IISPH context: call sph_set_iisph(1) before it "
    "(WCSPH contexts use sph_shard_configure_bodies; dynamic solids in DFSPH are single-GPU)";
const char *const kShardBodiesFixed =
    "the body table of a context configured by sph_shard_configure_bodies is fixed: configure a new context";
const char *const kNoDfsph = "sph_set_dfsph(1) was not called";
const char *const kNoIisph = "sph_set_iisph(1) was not called";
const char *const kPcisphContext =
    "this context is in PCISPH mode (sph_set_pcisph): it steps with sph_pcisph_op / sph_pcisph_solve / sph_pcisph_step";
// sph_shard_configure and the body configures refuse a PCISPH context, and sph_set_pcisph(1) a sharded one: a PCISPH
// context shards through sph_shard_configure_pcisph only, in PCISPH mode from the start
const char *const kPcisphSingleGpu =
    "PCISPH (sph_set_pcisph) is single-GPU: x-slab sharding runs WCSPH, DFSPH and IISPH contexts";
const char *const kNoPcisph = "sph_set_pcisph(1) was not called";
// sharded PCISPH (sph_shard_pcisph_step) runs fluid and static solids; the single-GPU PCISPH calls launch over the
// capacity of a sharded context and would step its ghost and trash records too
const char *const kPcisphSharded = "this PCISPH context is sharded: step it with sph_shard_pcisph_step";
const char *const kPcisphShardStep =
    "this context is in PCISPH mode (sph_set_pcisph): a sharded PCISPH context steps with sph_shard_pcisph_step";
const char *const kShardPcisphContext =
    "sph_shard_configure_pcisph shards a PCISPH context: call sph_set_pcisph(1) before it (WCSPH, DFSPH and IISPH "
    "contexts use sph_shard_configure)";
const char *const kShardBodiesPcisph =
    "x-slab sharding of a PCISPH context runs fluid and static solids: dynamic solids in PCISPH are single-GPU";
const char *const kWorldChanged = "the transport's world size changed after sph_shard_configure: configure again";
// device copy P.dfsph, set for IISPH and PCISPH too: the three list-based solvers share the density pass (no clamp,
// no EOS)
enum class Solver { WCSPH, DFSPH, IISPH, PCISPH };
// device copy P.slab_on; Static: sph_shard_configure, Bodies: sph_shard_configure_bodies / _iisph_bodies
enum class ShardMode { Off, Static, Bodies };

constexpr int NUM_TIMERS = 12;
constexpr int GRAPH_UNROLL = 4;  // must be even (ping-pong parity returns to its start)
const char *kTimerNames[NUM_TIMERS] = {"zero",  "hash",    "scan",  "bucket",    "rank_move", "boundary_volume",
                                       "density", "force", "advect_clamp", "rigid", "unused",    "total"};
enum { T_ZERO, T_HASH, T_SCAN, T_BUCKET, T_MOVE, T_BVOL, T_DENSITY, T_FORCE, T_ADVECT, T_RIGID, T_UNUSED, T_TOTAL };

inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

struct Layout {
    uint64_t off_state[14];  // posm, veld, x0id, misc, acc (x2), aux, fpv (2 slots, contiguous), dfs
    uint64_t off_cid, off_grid_ids, off_perm, off_ticket;
    uint64_t off_zero_begin, off_tile_counter, off_tile_state, off_cell_end, off_zero_end;
    uint64_t off_solid_slot, off_status, off_bodies, off_scratch, off_nbr_list, off_nbr_cnt;
    int64_t npad;
    uint64_t total;
    int n_tiles;
};

Layout make_layout(int64_t n_max, int64_t C, int64_t n_solid, int n_bodies) {
    Layout L;
    uint64_t o = 0;
    auto take = [&](uint64_t bytes) { uint64_t r = o; o = align_up(o + bytes, 256); return r; };
    uint64_t n = (uint64_t)(n_max > 0 ? n_max : 1);
    for (int k = 0; k < 14; ++k) {
        if (k == 12) { L.off_state[k] = L.off_state[11] + n * sizeof(float4); continue; }  // second half of fpv
        L.off_state[k] = take((k == 11 ? 2 : 1) * n * sizeof(float4));
    }
    L.off_cid = take(n * 4);
    L.off_grid_ids = take(n * 4);
    L.off_perm = take(n * 4);
    L.off_ticket = take(n * 4);
    L.n_tiles = (int)((C + 1 + SCAN_TILE - 1) / SCAN_TILE);  // +1: the slab-mode trash bucket
    // one contiguous region that a single memset clears every build
    L.off_zero_begin = o;
    L.off_tile_counter = take(256);
    L.off_tile_state = take((uint64_t)L.n_tiles * 8);
    L.off_cell_end = take((uint64_t)(C + 1) * 4);
    L.off_zero_end = o;
    L.off_solid_slot = take((uint64_t)(n_solid > 0 ? n_solid : 1) * 4);
    L.off_status = take(256);
    L.off_bodies = take((uint64_t)(n_bodies > 0 ? n_bodies : 1) * sizeof(RigidBodyDev));
    L.off_scratch = take(256);
    L.npad = (int64_t)align_up(n, 32);
    L.off_nbr_cnt = take((uint64_t)L.npad * 4);
    L.off_nbr_list = take((uint64_t)L.npad * 4 * NBR_CAP);
    L.total = o;
    return L;
}

constexpr uint64_t SHARD_HDR_BYTES = 64;  // the 16-int header that travels with every record exchange

// The shard buffer (library-owned, x-slab sharding): {device step state | send header x 2 | 2 sides x 4 send staging
// arrays x halo_cap records | sharded DFSPH: DX ranges + alignment headers | one fp64 error partial per rank
// [| with shape-matched bodies: every rank's table of the body particles' records, 2 x 16 bytes per body particle]}
struct ShardLayout {
    uint64_t off_state, off_hdr[2], off_stage[2][4], off_dx, off_err, off_body;
    uint64_t total;
};

ShardLayout make_shard_layout(int64_t halo_cap, int world, int64_t n_body_particles = 0) {
    ShardLayout L;
    uint64_t o = 0;
    auto take = [&](uint64_t bytes) { uint64_t r = o; o = align_up(o + bytes, 256); return r; };
    L.off_state = take(SD_INTS * 4);
    for (int side = 0; side < 2; ++side) L.off_hdr[side] = take(SHARD_HDR_BYTES);
    for (int side = 0; side < 2; ++side)
        for (int k = 0; k < 4; ++k) L.off_stage[side][k] = take((uint64_t)halo_cap * 16);
    L.off_dx = take(DX_INTS * 4);
    L.off_err = take((uint64_t)world * 8);
    L.off_body = n_body_particles > 0 ? take((uint64_t)world * n_body_particles * 32) : 0;
    L.total = o;
    return L;
}

struct GraphSlot {  // one instantiated CUDA graph and the kernels a replay of it launches
    cudaGraphExec_t exec = nullptr;
    int64_t kernels = 0;
};

#ifndef SPH_EMU
// NCCL point-to-point through dlopen: the library has no link-time dependency on NCCL (the CPU test-suite and
// single-GPU users never load it); inside a PyTorch process the already loaded libnccl.so.2 is reused.
struct NcclId { char internal[128]; };
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(NcclId *) = nullptr;
    int (*CommInitRank)(void **, int, NcclId, int) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    std::string err;
};
NcclApi g_nccl;
bool load_nccl() {
    if (g_nccl.lib) return true;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { g_nccl.err = std::string("cannot load libnccl.so.2: ") + dlerror(); return false; }
    auto sym = [&](const char *n) { void *p = dlsym(h, n); if (!p) g_nccl.err = std::string("libnccl lacks ") + n; return p; };
    g_nccl.GetUniqueId = reinterpret_cast<int (*)(NcclId *)>(sym("ncclGetUniqueId"));
    g_nccl.CommInitRank = reinterpret_cast<int (*)(void **, int, NcclId, int)>(sym("ncclCommInitRank"));
    g_nccl.CommDestroy = reinterpret_cast<int (*)(void *)>(sym("ncclCommDestroy"));
    g_nccl.GroupStart = reinterpret_cast<int (*)()>(sym("ncclGroupStart"));
    g_nccl.GroupEnd = reinterpret_cast<int (*)()>(sym("ncclGroupEnd"));
    g_nccl.Send = reinterpret_cast<int (*)(const void *, size_t, int, int, void *, cudaStream_t)>(sym("ncclSend"));
    g_nccl.Recv = reinterpret_cast<int (*)(void *, size_t, int, int, void *, cudaStream_t)>(sym("ncclRecv"));
    g_nccl.GetErrorString = reinterpret_cast<const char *(*)(int)>(sym("ncclGetErrorString"));
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.GroupStart || !g_nccl.GroupEnd ||
        !g_nccl.Send || !g_nccl.Recv || !g_nccl.GetErrorString)
        return false;
    g_nccl.lib = h;
    return true;
}
#endif

}  // namespace

struct SphCtx {
    SphParams hp;
    DevParams P;
    DevArrays S;
    Layout L;
    int device = 0;
    int sms = 1;  // multiprocessors of `device` (sizes the grid-stride grids of sharded steps)
    int64_t n_max = 0, n_solid_cap = 0;
    int body_cap = 0;
    char *ws = nullptr;
    std::vector<SphRigidBody> bodies;
    bool has_dynamic_solids = true;  // conservative until pack() inspects the flags
    std::string err;
    int64_t launches = 0;
    // CUDA graphs, one per ping-pong parity
    GraphSlot graph[2];
    GraphSlot graph_multi[2];  // GRAPH_UNROLL steps per replay
    int parity = 0;
    bool time_pair = false;
    cudaEvent_t pair_ev[3] = {nullptr, nullptr, nullptr};
    cudaStream_t capture_stream = nullptr;  // graphs are captured here (the legacy stream cannot capture)
    bool built = false;  // neighbour structure valid for current positions
    bool list_valid = false;  // neighbour lists valid for current positions (DFSPH kernels)
    Solver solver = Solver::WCSPH;  // written by set_solver only, together with P.dfsph
    // x-slab sharding (sph_shard_*)
    SphTransport transport{};
    bool has_transport = false;
    int rank = 0, world = 1;
    void *nccl_comm = nullptr;
    char *shard_buf = nullptr;  // library-owned: device step state + send staging (cudaMalloc at sph_shard_configure)
    ShardLayout SL{};
    bool shard_begun = false;
    cudaStream_t comm_stream = nullptr;
    cudaEvent_t ev_packed = nullptr, ev_exchanged = nullptr;
    GraphSlot graph_shard[2][2];  // [parity][wide exchange]
    int32_t narrow_cap = 0;      // records per side of the usual (sgw + 1 layers) exchange; halo_cap = sgw + 2 layers
    // hide the exchange behind the interior densities too (boundary densities first): meant for a rank that talks to
    // two neighbours, whose exchange can outlast the interior force pass; with one neighbour or short exchanges the
    // second density launch can cost more than it hides (not measured on H100s)
    bool split_density = false;
    int64_t shard_sequences = 0;  // sequences run so far (begin = 0): sequence q feeds the plan kernel of q + 1
    // sharded DFSPH: records per side of the ghost alignment (sgw layers) and of a per-sweep exchange (one layer)
    int32_t align_cap = 0, sweep_cap = 0;
    int shard_world = 1;  // world size the shard buffer's per-rank error partials and body tables were sized for
    // Bodies: a WCSPH context steps with shard_bodies_sequence, an IISPH one with shard_dfsph_sequence's body hooks
    ShardMode shard = ShardMode::Off;  // set by shard_setup and shard_configure_bodies, together with P.slab_on
    uint64_t xfer_groups = 0, xfer_bytes = 0;  // transport groups issued from the host, and the bytes this rank sent
    // sph_shard_dump's device scratch (library-owned, grown on demand): the header sent, the headers received, the
    // tile counts
    char *dump_buf = nullptr;
    uint64_t dump_bytes = 0;
};

namespace {

int fail(SphCtx *ctx, int code, const std::string &msg) {
    if (ctx) ctx->err = msg; else g_create_error = msg;
    return code;
}

// What an entry point needs of a context's solver and shard mode.  A NULL refusal message means no such requirement;
// the messages that differ between entry points are the entry point's own.
struct Need {
    bool configured = false, begun = false, grid = false, lists = false;
    Solver solver = Solver::WCSPH;
    const char *other_solver = nullptr, *if_sharded = nullptr, *if_bodies = nullptr, *if_moved = nullptr;
    Need &sharded() { configured = true; return *this; }
    Need &runs(Solver s, const char *refusal) { solver = s; other_solver = refusal; return *this; }
    Need &shard_step(Solver s, const char *refusal) { configured = begun = true; return runs(s, refusal); }
    Need &unsharded(const char *refusal) { if_sharded = refusal; return *this; }
    Need &no_bodies(const char *refusal) { if_bodies = refusal; return *this; }
    Need &same_world(const char *refusal) { if_moved = refusal; return *this; }
    Need &built() { grid = true; return *this; }  // neighbour structure valid, unless there are no particles
    Need &fresh_lists() { lists = true; return *this; }  // neighbour lists valid too
};

// The mode checks of every entry point, in this order: configured, the entry point's bare argument checks (args_ok),
// solver, not sharded, not a body context, begun, world size unchanged, then the neighbour structure; returns the first
// refusal or SPH_OK.  Other solvers' entry points refuse an IISPH or a PCISPH context with one message per kind (sharded
// or not).
int require(SphCtx *c, const Need &n, bool args_ok = true) {
    if (!c) return SPH_E_ARG;
    if (n.configured && c->shard == ShardMode::Off) return fail(c, SPH_E_ARG, "sph_shard_configure was not called");
    if (!args_ok) return SPH_E_ARG;
    if (n.other_solver && c->solver != n.solver)
        return fail(c, SPH_E_ARG, c->solver == Solver::IISPH    ? (n.configured ? kIisphShardStep : kIisphContext)
                                  : c->solver == Solver::PCISPH ? (n.configured ? kPcisphShardStep : kPcisphContext)
                                                                : n.other_solver);
    if (n.if_sharded && c->shard != ShardMode::Off) return fail(c, SPH_E_ARG, n.if_sharded);
    if (n.if_bodies && c->shard == ShardMode::Bodies) return fail(c, SPH_E_ARG, n.if_bodies);
    if (n.begun && !c->shard_begun) return fail(c, SPH_E_ARG, "sph_shard_begin was not called");
    if (n.if_moved && c->world != c->shard_world) return fail(c, SPH_E_ARG, n.if_moved);
    if (n.grid && c->P.n > 0 && !c->built)
        return fail(c, SPH_E_ARG, "neighbour structure is stale: call sph_neighbor_build first (the reference's kernels "
                                  "would read an outdated grid here)");
    if (n.lists && (!c->built || !c->list_valid))
        return fail(c, SPH_E_ARG, "neighbour lists are stale: run sph_neighbor_build and op 0 (compute_densities) first");
    return SPH_OK;
}

#define CUDA_TRY(ctx, expr)                                                                        \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail((ctx), SPH_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));    \
    } while (0)

int validate_params(const SphParams *p, std::string &why) {
    if (!p) { why = "params is NULL"; return SPH_E_ARG; }
    if (p->dim != 3) { why = "only dim == 3 is supported (2-D is unreachable in the reference)"; return SPH_E_ARG; }
    for (int a = 0; a < 3; ++a)
        if (p->grid_num[a] < 3) { why = "grid_num must be >= 3 per axis"; return SPH_E_ARG; }
    if (!(p->h > 0.f) || !(p->density0 > 0.f)) { why = "h and density0 must be positive"; return SPH_E_ARG; }
    int64_t C = (int64_t)p->grid_num[0] * p->grid_num[1] * p->grid_num[2];
    if (C >= (1ll << 31)) { why = "too many grid cells for int32 indices"; return SPH_E_CAPACITY; }
    return SPH_OK;
}

void derive_params(SphCtx *c) { derive_dev_params(c->P, c->hp); }

void bind_arrays(SphCtx *c) {
    char *w = c->ws;
    const Layout &L = c->L;
    DevArrays &S = c->S;
    float4 *st[14];
    for (int k = 0; k < 14; ++k) st[k] = reinterpret_cast<float4 *>(w + L.off_state[k]);
    int p = c->parity;
    S.posm = st[0 + 5 * p]; S.veld = st[1 + 5 * p]; S.x0id = st[2 + 5 * p]; S.misc = st[3 + 5 * p]; S.acc = st[4 + 5 * p];
    int q = 1 - p;
    S.posm_n = st[0 + 5 * q]; S.veld_n = st[1 + 5 * q]; S.x0id_n = st[2 + 5 * q]; S.misc_n = st[3 + 5 * q]; S.acc_n = st[4 + 5 * q];
    S.aux = st[10];
    S.fpv = st[11];  // 2 float4 per particle
    S.dfs = st[13];
    S.cid = reinterpret_cast<int32_t *>(w + L.off_cid);
    S.grid_ids = reinterpret_cast<int32_t *>(w + L.off_grid_ids);
    S.perm = reinterpret_cast<int32_t *>(w + L.off_perm);
    S.tile_counter = reinterpret_cast<int32_t *>(w + L.off_tile_counter);
    S.tile_state = reinterpret_cast<unsigned long long *>(w + L.off_tile_state);
    S.cell_end = reinterpret_cast<int32_t *>(w + L.off_cell_end);
    S.ticket = reinterpret_cast<int32_t *>(w + L.off_ticket);
    S.solid_slot = reinterpret_cast<int32_t *>(w + L.off_solid_slot);
    S.status = reinterpret_cast<uint32_t *>(w + L.off_status);
    S.nbr_list = reinterpret_cast<int32_t *>(w + L.off_nbr_list);
    S.nbr_cnt = reinterpret_cast<int32_t *>(w + L.off_nbr_cnt);
    S.npad = (int32_t)L.npad;
    S.sd = nullptr;
    if (c->shard_buf) {
        S.sd = reinterpret_cast<int32_t *>(c->shard_buf + c->SL.off_state);
        for (int side = 0; side < 2; ++side) {
            S.stage_hdr[side] = reinterpret_cast<int32_t *>(c->shard_buf + c->SL.off_hdr[side]);
            for (int k = 0; k < 4; ++k) S.stage[side][k] = reinterpret_cast<float4 *>(c->shard_buf + c->SL.off_stage[side][k]);
        }
    }
}

inline RigidBodyDev *dev_bodies(SphCtx *c) { return reinterpret_cast<RigidBodyDev *>(c->ws + c->L.off_bodies); }
int store_bodies(SphCtx *ctx, const SphRigidBody *bodies, int32_t n_bodies);

inline int blocks_for(int64_t n, int t) { return (int)((n + t - 1) / t); }
// Sharded steps: n is the capacity and the real counts are device state, so the LIGHT step kernels (histogram,
// bucket, rank + move) run grid-stride loops over the compact input numbering on a grid of `per_sm` resident blocks
// per SM instead of one thread per capacity slot; the pair kernels keep one block per tile.
inline int step_grid(const SphCtx *c, int64_t n, int t, int per_sm) {
    const int full = blocks_for(n, t);
    return c->P.slab_on ? std::min(full, c->sms * per_sm) : full;
}

// Launch with programmatic stream serialisation (the kernels of the step chain start with pdl_wait()): the next
// kernel's blocks are scheduled while the previous grid drains, which hides most of the launch gap between graph
// nodes.  SPH_PDL=0 switches it off (A/B).
#ifdef SPH_EMU
#define PDL_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#else
const bool g_pdl = !(std::getenv("SPH_PDL") && std::atoi(std::getenv("SPH_PDL")) == 0);
template <typename... KArgs, typename... Args>
inline void pdl_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = g_pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#define PDL_LAUNCH(kern, grid, block, st, ...) pdl_launch(kern, dim3(grid), dim3(block), st, __VA_ARGS__)
#endif

void drop_graphs(SphCtx *c) {
    auto drop = [](GraphSlot &g) { if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; } };
    for (int k = 0; k < 2; ++k) {
        drop(c->graph[k]);
        drop(c->graph_multi[k]);
        for (int w = 0; w < 2; ++w) drop(c->graph_shard[k][w]);
    }
}

void set_solver(SphCtx *c, Solver s) { c->solver = s; c->P.dfsph = s != Solver::WCSPH; drop_graphs(c); }

// ---- launch sequences -----------------------------------------------------------------
struct StageTimer {
    cudaEvent_t ev[NUM_TIMERS + 1];
    int stage_of[NUM_TIMERS + 1];
    int count = 0;
    bool on = false;
    cudaStream_t st = nullptr;
    void mark(int stage) {
        if (!on) return;
        cudaEventCreate(&ev[count]);
        cudaEventRecord(ev[count], st);
        stage_of[count] = stage;
        ++count;
    }
};

// particle_system.py:372-375.  Kernel count returned through *kernels.
int launch_neighbor_build(SphCtx *c, cudaStream_t st, StageTimer *tm, int64_t *kernels, bool move_acc = true) {
    const DevParams &P = c->P;
    if (P.n == 0) return SPH_OK;
    const Layout &L = c->L;
    if (tm) tm->mark(T_ZERO);
    CUDA_TRY(c, cudaMemsetAsync(c->ws + L.off_zero_begin, 0, L.off_zero_end - L.off_zero_begin, st));
    if (tm) tm->mark(T_HASH);
    PDL_LAUNCH(k_hash_count, step_grid(c, P.n, 256, 8), 256, st, P, c->S);
    if (tm) tm->mark(T_SCAN);
    PDL_LAUNCH(k_scan, L.n_tiles, SCAN_THREADS, st, c->S.cell_end, P.C + 1, c->S.tile_state, c->S.tile_counter);
    if (tm) tm->mark(T_BUCKET);
    PDL_LAUNCH(k_bucket, step_grid(c, P.n, 256, 8), 256, st, P, c->S);
    if (tm) tm->mark(T_MOVE);
    if (move_acc) PDL_LAUNCH(k_rank_move<true>, step_grid(c, P.n, 256, 8), 256, st, P, c->S);
    else PDL_LAUNCH(k_rank_move<false>, step_grid(c, P.n, 256, 8), 256, st, P, c->S);
    *kernels += 4;
    CUDA_TRY(c, cudaGetLastError());
    c->parity ^= 1;  // sorted state now lives in the other buffer set
    bind_arrays(c);
    c->built = true;
    return SPH_OK;
}

// density + neighbour lists, then forces (+ integration).
// n_grid (sharded DFSPH): the grid covers [0, n_grid) instead of all P.n slots
void launch_pair_density(SphCtx *c, cudaStream_t st, int64_t *kernels, int split_mode = 0, int64_t n_grid = -1) {
    const DevParams &P = c->P;
    const int blocks = blocks_for(n_grid < 0 ? P.n : n_grid, DENS_WARPS * 32);
    if (P.dfsph) PDL_LAUNCH((k_density_tma<false>), blocks, DENS_WARPS * 32, st, P, c->S, split_mode);
    else PDL_LAUNCH((k_density_tma<true>), blocks, DENS_WARPS * 32, st, P, c->S, split_mode);
    *kernels += 1;
}
void launch_pair_force_and_advect(SphCtx *c, cudaStream_t st, StageTimer *tm, int64_t *kernels, int split_mode = 0) {
    const DevParams &P = c->P;
    if (P.uniform_fluid) {
        if (P.slab_on)
            PDL_LAUNCH((k_force_packed<FORCE_BATCH, FORCE_THREADS, true>), blocks_for(P.n, FORCE_THREADS), FORCE_THREADS, st, P,
                       c->S, split_mode);
        else
            PDL_LAUNCH((k_force_packed<FORCE_BATCH, FORCE_THREADS>), blocks_for(P.n, FORCE_THREADS), FORCE_THREADS, st, P, c->S,
                       split_mode);
        *kernels += 1;
        if (tm) tm->mark(T_ADVECT);
        if (c->has_dynamic_solids && P.n_solid > 0) {
            k_advect_solids<<<blocks_for(P.n_solid, 256), 256, 0, st>>>(P, c->S);
            *kernels += 1;
        }
        return;
    }
    k_force_general<4, 128><<<blocks_for(P.n, 128), 128, 0, st>>>(P, c->S);
    if (tm) tm->mark(T_ADVECT);
    k_advect<true><<<blocks_for(P.n, 256), 256, 0, st>>>(P, c->S);
    *kernels += 2;
}

int launch_boundary_volume(SphCtx *c, int moving, cudaStream_t st, int64_t *kernels) {
    const DevParams &P = c->P;
    if (P.n_solid == 0) return SPH_OK;
    k_boundary_volume<false><<<blocks_for((int64_t)P.n_solid * 32, 128), 128, 0, st>>>(P, c->S, moving);
    *kernels += 1;
    CUDA_TRY(c, cudaGetLastError());
    return SPH_OK;
}

int launch_rigid_solve(SphCtx *c, cudaStream_t st, int64_t *kernels) {
    // sph_base.py:247-260: per dynamic body solve_constraints, then enforce_boundary_3D(solid) -- all bodies in ONE
    // launch (one CTA per body carries the clamps of the whole loop for its own particles, see k_rigid), the dynamic
    // solids outside every body in a second one
    const int nb = (int)c->bodies.size();
    if (nb == 0) return SPH_OK;
    k_rigid<<<nb, RIGID_THREADS, 0, st>>>(c->P, c->S, dev_bodies(c), 0, 2, nullptr, nb);
    k_enforce_boundary_solid<false><<<blocks_for(c->P.n_solid, 256), 256, 0, st>>>(c->P, c->S, nb, dev_bodies(c), nb);
    *kernels += 2;
    CUDA_TRY(c, cudaGetLastError());
    return SPH_OK;
}

// One whole SPHBase.step() with the fused kernels (sph_base.py:263-271, WCSPH.py:152-156).
int launch_step(SphCtx *c, cudaStream_t st, StageTimer *tm, int64_t *kernels) {
    const DevParams &P = c->P;
    if (P.n == 0) return SPH_OK;
    int rc = launch_neighbor_build(c, st, tm, kernels, /*move_acc=*/false);
    if (rc) return rc;
    if (tm) tm->mark(T_BVOL);
    if (c->has_dynamic_solids) { rc = launch_boundary_volume(c, 1, st, kernels); if (rc) return rc; }
    if (tm) tm->mark(T_DENSITY);
    launch_pair_density(c, st, kernels);
    if (tm) tm->mark(T_FORCE);
    launch_pair_force_and_advect(c, st, tm, kernels);
    if (tm) tm->mark(T_RIGID);
    if (!c->bodies.empty()) { rc = launch_rigid_solve(c, st, kernels); if (rc) return rc; }
    if (tm) tm->mark(T_TOTAL);
    CUDA_TRY(c, cudaGetLastError());
    c->built = false; c->list_valid = false;  // positions moved
    return SPH_OK;
}

// Replay the graph in `slot`, capturing it first if the slot is empty: issue(stream, kernels) launches `span`
// consecutive steps starting from the current ping-pong parity.  `what` names the graph in error messages.
template <typename Issue>
int replay_graph(SphCtx *ctx, cudaStream_t st, GraphSlot &slot, int span, cudaStreamCaptureMode mode, const char *what,
                 Issue issue) {
    const int par = ctx->parity;
    if (!slot.exec) {
        cudaGraph_t g = nullptr;
        int64_t kernels = 0;
        if (!ctx->capture_stream) CUDA_TRY(ctx, cudaStreamCreateWithFlags(&ctx->capture_stream, cudaStreamNonBlocking));
        cudaStream_t cs = ctx->capture_stream;
        CUDA_TRY(ctx, cudaStreamBeginCapture(cs, mode));
        const int rc = issue(cs, &kernels);
        cudaError_t e = cudaStreamEndCapture(cs, &g);
        // capture advanced the host-side parity exactly as real steps do; rewind
        ctx->parity = par;
        bind_arrays(ctx);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) return fail(ctx, SPH_E_CUDA, std::string(what) + " capture: " + cudaGetErrorString(e));
        e = cudaGraphInstantiate(&slot.exec, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(ctx, SPH_E_CUDA, std::string(what) + " instantiate: " + cudaGetErrorString(e));
        slot.kernels = kernels;
    }
    CUDA_TRY(ctx, cudaGraphLaunch(slot.exec, st));
    ctx->launches += slot.kernels;
    if (span & 1) { ctx->parity = par ^ 1; bind_arrays(ctx); }
    ctx->built = false; ctx->list_valid = false;  // positions moved
    return SPH_OK;
}

}  // namespace

// =========================================================================================
// extern "C" ABI
// =========================================================================================
extern "C" {

uint64_t sph_workspace_bytes(const SphParams *params, int64_t n_max, int64_t n_solid, int32_t n_bodies) {
    std::string why;
    if (validate_params(params, why) != SPH_OK || n_max < 0 || n_solid < 0 || n_bodies < 0) return 0;
    int64_t C = (int64_t)params->grid_num[0] * params->grid_num[1] * params->grid_num[2];
    return make_layout(n_max, C, n_solid, n_bodies).total;
}

int sph_create(const SphParams *params, int64_t n_max, int64_t n_solid, int32_t n_bodies, int32_t device,
               void *workspace, uint64_t workspace_bytes, SphCtx **out) {
    if (!out) return fail(nullptr, SPH_E_ARG, "out is NULL");
    *out = nullptr;
    std::string why;
    int rc = validate_params(params, why);
    if (rc) return fail(nullptr, rc, why);
    if (n_max < 0 || n_max >= (1ll << 31) - 1) return fail(nullptr, SPH_E_CAPACITY, "n_max out of int32 range");
    if ((uint64_t)align_up((uint64_t)(n_max > 0 ? n_max : 1), 32) * (uint64_t)NBR_CAP >= (1ull << 32))
        return fail(nullptr, SPH_E_CAPACITY, "n_max too large: neighbour-list slots are 32-bit (NBR_CAP * n_max < 2^32)");
    if (n_solid < 0 || n_bodies < 0) return fail(nullptr, SPH_E_ARG, "negative capacity");
    if (!workspace) return fail(nullptr, SPH_E_ARG, "workspace is NULL");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(nullptr, SPH_E_ARG, "workspace must be 256-byte aligned");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, SPH_E_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") + cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(nullptr, SPH_E_ARG, "device index out of range");
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(nullptr, SPH_E_CUDA, cudaGetErrorString(e));
    SphCtx *c = new (std::nothrow) SphCtx();
    if (!c) return fail(nullptr, SPH_E_CAPACITY, "out of host memory");
    c->hp = *params;
    c->device = device;
    e = cudaDeviceGetAttribute(&c->sms, cudaDevAttrMultiProcessorCount, device);
    if (e != cudaSuccess) { delete c; return fail(nullptr, SPH_E_CUDA, cudaGetErrorString(e)); }
    c->n_max = n_max;
    c->n_solid_cap = n_solid;
    c->body_cap = n_bodies;
    int64_t C = (int64_t)params->grid_num[0] * params->grid_num[1] * params->grid_num[2];
    c->L = make_layout(n_max, C, n_solid, n_bodies);
    if (c->L.total > workspace_bytes) { delete c; return fail(nullptr, SPH_E_CAPACITY, "workspace too small"); }
    c->ws = static_cast<char *>(workspace);
    c->P = DevParams{};
    derive_params(c);
    c->P.n = 0;
    c->P.n_solid = 0;
    bind_arrays(c);
    e = cudaMemset(c->ws + c->L.off_status, 0, 256);
    if (e != cudaSuccess) { std::string m = cudaGetErrorString(e); delete c; return fail(nullptr, SPH_E_CUDA, m); }
    *out = c;
    return SPH_OK;
}

int sph_destroy(SphCtx *ctx) {
    if (!ctx) return SPH_OK;
    drop_graphs(ctx);
    if (ctx->capture_stream) cudaStreamDestroy(ctx->capture_stream);
#ifndef SPH_EMU
    if (ctx->nccl_comm && g_nccl.lib) g_nccl.CommDestroy(ctx->nccl_comm);
    if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
    if (ctx->ev_packed) cudaEventDestroy(ctx->ev_packed);
    if (ctx->ev_exchanged) cudaEventDestroy(ctx->ev_exchanged);
#endif
    if (ctx->shard_buf) cudaFree(ctx->shard_buf);
    if (ctx->dump_buf) cudaFree(ctx->dump_buf);
    delete ctx;
    return SPH_OK;
}

const char *sph_last_error(const SphCtx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int sph_set_params(SphCtx *ctx, const SphParams *params) {
    if (!ctx) return SPH_E_ARG;
    std::string why;
    int rc = validate_params(params, why);
    if (rc) return fail(ctx, rc, why);
    for (int a = 0; a < 3; ++a)
        if (params->grid_num[a] != ctx->hp.grid_num[a]) return fail(ctx, SPH_E_ARG, "grid_num cannot change after creation");
    ctx->hp = *params;
    int n = ctx->P.n, ns = ctx->P.n_solid;
    derive_params(ctx);
    ctx->P.n = n; ctx->P.n_solid = ns;
    drop_graphs(ctx);
    return SPH_OK;
}

int sph_pack(SphCtx *ctx, const SphFields *f, int64_t n, void *stream) {
    if (!ctx || !f) return SPH_E_ARG;
    if (n < 0 || n > ctx->n_max) return fail(ctx, SPH_E_CAPACITY, "particle count exceeds n_max");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ctx->P.n = (int32_t)n;
    drop_graphs(ctx);
    ctx->built = false; ctx->list_valid = false;
    if (n == 0) return SPH_OK;
    k_pack<<<blocks_for(n, 256), 256, 0, st>>>(ctx->P, ctx->S, *f);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_set_solid_count(SphCtx *ctx, int64_t n_solid, int32_t has_dynamic_solids) {
    if (!ctx) return SPH_E_ARG;
    if (n_solid < 0 || n_solid > ctx->n_solid_cap) return fail(ctx, SPH_E_CAPACITY, "n_solid exceeds the capacity given at creation");
    if (int rc = require(ctx, Need().unsharded(n_solid > 0 && has_dynamic_solids ? kShardStaticOnly : nullptr))) return rc;
    ctx->P.n_solid = (int32_t)n_solid;
    ctx->has_dynamic_solids = has_dynamic_solids != 0;
    drop_graphs(ctx);
    return SPH_OK;
}

int sph_set_fluid_uniform(SphCtx *ctx, int32_t uniform, float fluid_m, float fluid_mV) {
    if (!ctx) return SPH_E_ARG;
    ctx->P.uniform_fluid = uniform ? 1 : 0;
    ctx->P.fluid_m = fluid_m;
    ctx->P.fluid_mV = fluid_mV;
    drop_graphs(ctx);
    return SPH_OK;
}

int sph_unpack(SphCtx *ctx, const SphFields *f, void *stream) {
    if (!ctx || !f) return SPH_E_ARG;
    if (ctx->P.n == 0) return SPH_OK;
    k_unpack<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, *f);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_unpack_xv(SphCtx *ctx, float *x, float *v, int32_t *object_id, void *stream) {
    if (!ctx || !x || !v) return SPH_E_ARG;
    if (ctx->P.n == 0) return SPH_OK;
    k_unpack_xv<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, x, v, object_id);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_upload_xv(SphCtx *ctx, const float *x, const float *v, void *stream) {
    if (!ctx || !x || !v) return SPH_E_ARG;
    if (ctx->P.n == 0) return SPH_OK;
    k_upload_xv<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, x, v);
    ctx->launches += 1;
    ctx->built = false; ctx->list_valid = false;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_copy_grid_particles_num(SphCtx *ctx, int32_t *out_dev, void *stream) {
    if (!ctx || !out_dev) return SPH_E_ARG;
    CUDA_TRY(ctx, cudaMemcpyAsync(out_dev, ctx->S.cell_end, (size_t)ctx->P.C * 4, cudaMemcpyDeviceToDevice,
                                  static_cast<cudaStream_t>(stream)));
    return SPH_OK;
}

int sph_neighbor_build(SphCtx *ctx, void *stream) {
    if (!ctx) return SPH_E_ARG;
    return launch_neighbor_build(ctx, static_cast<cudaStream_t>(stream), nullptr, &ctx->launches);
}

int sph_boundary_volume(SphCtx *ctx, int32_t moving, void *stream) {
    if (int rc = require(ctx, Need().unsharded(kShardStaticOnly).built())) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    return launch_boundary_volume(ctx, moving, static_cast<cudaStream_t>(stream), &ctx->launches);
}

int sph_compute_densities(SphCtx *ctx, void *stream) {
    if (int rc = require(ctx, Need().built())) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    k_density_simple<<<blocks_for(ctx->P.n, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_compute_non_pressure_forces(SphCtx *ctx, void *stream) {
    if (int rc = require(ctx, Need().built())) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    k_force_simple<true, false><<<blocks_for(ctx->P.n, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_compute_pressure_forces(SphCtx *ctx, void *stream) {
    if (int rc = require(ctx, Need().built())) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    k_eos<<<blocks_for(ctx->P.n, 256), 256, 0, st>>>(ctx->P, ctx->S);
    k_force_simple<false, true><<<blocks_for(ctx->P.n, 128), 128, 0, st>>>(ctx->P, ctx->S);
    ctx->launches += 2;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_advect(SphCtx *ctx, void *stream) {
    if (!ctx) return SPH_E_ARG;
    if (ctx->P.n == 0) return SPH_OK;
    k_advect<false><<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S);
    ctx->launches += 1;
    ctx->built = false; ctx->list_valid = false;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_enforce_boundary(SphCtx *ctx, int32_t particle_type, void *stream) {
    if (!ctx) return SPH_E_ARG;
    if (ctx->P.n == 0) return SPH_OK;
    k_enforce_boundary<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, particle_type);
    ctx->launches += 1;
    ctx->built = false; ctx->list_valid = false;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_set_rigid_bodies(SphCtx *ctx, const SphRigidBody *bodies, int32_t n_bodies) {
    if (!ctx || n_bodies < 0 || (n_bodies > 0 && !bodies)) return SPH_E_ARG;
    if (n_bodies > ctx->body_cap) return fail(ctx, SPH_E_CAPACITY, "more rigid bodies than the workspace was sized for");
    if (int rc = require(ctx, Need().unsharded(n_bodies > 0 ? kShardStaticOnly : nullptr).no_bodies(kShardBodiesFixed))) return rc;
    for (int b = 0; b < n_bodies; ++b)  // validate everything before any state changes
        if (bodies[b].solid_begin < 0 || bodies[b].solid_end < bodies[b].solid_begin || bodies[b].solid_end > ctx->n_solid_cap)
            return fail(ctx, SPH_E_ARG, "rigid body solid-id range out of bounds");
    return store_bodies(ctx, bodies, n_bodies);
}

}  // extern "C"
namespace {
// The body table on the host and on the device (R = I, cm = 0 until the first solve).
int store_bodies(SphCtx *ctx, const SphRigidBody *bodies, int32_t n_bodies) {
    ctx->bodies.assign(bodies, bodies + n_bodies);
    std::vector<RigidBodyDev> h(n_bodies);
    for (int b = 0; b < n_bodies; ++b) {
        std::memset(&h[b], 0, sizeof(RigidBodyDev));
        h[b].object_id = bodies[b].object_id;
        h[b].solid_begin = bodies[b].solid_begin;
        h[b].solid_end = bodies[b].solid_end;
        for (int k = 0; k < 3; ++k) h[b].rest_cm[k] = bodies[b].rest_cm[k];
        h[b].R[0] = h[b].R[4] = h[b].R[8] = 1.0f;
    }
    if (n_bodies) CUDA_TRY(ctx, cudaMemcpy(dev_bodies(ctx), h.data(), sizeof(RigidBodyDev) * n_bodies, cudaMemcpyHostToDevice));
    drop_graphs(ctx);
    return SPH_OK;
}
}  // namespace
extern "C" {

static int rigid_call(SphCtx *ctx, int32_t body, int mode, float *out, void *stream) {
    if (int rc = require(ctx, Need().unsharded(kShardStaticOnly))) return rc;
    if (body < 0 || body >= (int)ctx->bodies.size()) return fail(ctx, SPH_E_ARG, "rigid body index out of range");
    k_rigid<<<1, RIGID_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, dev_bodies(ctx), body, mode, out, 0);
    ctx->launches += 1;
    if (mode == 2) { ctx->built = false; ctx->list_valid = false; }  // modes 0 / 1 only read
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_compute_com(SphCtx *ctx, int32_t body, float *out_dev, void *stream) {
    if (!out_dev) return SPH_E_ARG;
    return rigid_call(ctx, body, 0, out_dev, stream);
}
int sph_compute_rigid_rest_cm(SphCtx *ctx, int32_t body, void *stream) { return rigid_call(ctx, body, 1, nullptr, stream); }
int sph_solve_constraints(SphCtx *ctx, int32_t body, float *R_out_dev, void *stream) {
    return rigid_call(ctx, body, 2, R_out_dev, stream);
}

int sph_get_rigid_state(SphCtx *ctx, int32_t body, float *out_dev12, void *stream) {
    if (!ctx || !out_dev12) return SPH_E_ARG;
    if (body < 0 || body >= (int)ctx->bodies.size()) return fail(ctx, SPH_E_ARG, "rigid body index out of range");
    const RigidBodyDev *B = dev_bodies(ctx) + body;
    CUDA_TRY(ctx, cudaMemcpyAsync(out_dev12, B->R, sizeof(float) * 12, cudaMemcpyDeviceToDevice,
                                  static_cast<cudaStream_t>(stream)));  // R[9] and cm[3] are adjacent
    return SPH_OK;
}

int sph_step(SphCtx *ctx, int32_t nsteps, void *stream) {
    const char *dfsph = "sph_step is the fused WCSPH step; DFSPH is driven through sph_dfsph_op";
    if (int rc = require(ctx, Need().runs(Solver::WCSPH, dfsph), nsteps >= 0)) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int s = 0;
    while (s < nsteps) {
        // GRAPH_UNROLL (even) steps per replay amortise the graph-launch gap; the parity returns to its start
        const bool multi = nsteps - s >= GRAPH_UNROLL;
        const int span = multi ? GRAPH_UNROLL : 1;
        GraphSlot &slot = multi ? ctx->graph_multi[ctx->parity] : ctx->graph[ctx->parity];
        int rc = replay_graph(ctx, st, slot, span, cudaStreamCaptureModeThreadLocal, "graph",
                              [&](cudaStream_t cs, int64_t *kernels) {
                                  int rc = SPH_OK;
                                  for (int k = 0; k < span && rc == SPH_OK; ++k) rc = launch_step(ctx, cs, nullptr, kernels);
                                  return rc;
                              });
        if (rc) return rc;
        s += span;
    }
    return SPH_OK;
}

int sph_state_offsets(SphCtx *ctx, uint64_t *out5) {
    if (!ctx || !out5) return SPH_E_ARG;
    const float4 *cur[5] = {ctx->S.posm, ctx->S.veld, ctx->S.x0id, ctx->S.misc, ctx->S.acc};
    for (int k = 0; k < 5; ++k) out5[k] = (uint64_t)(reinterpret_cast<const char *>(cur[k]) - ctx->ws);
    return SPH_OK;
}

// =========================================================================================
// x-slab sharding (see include/sph_b200.h)
// =========================================================================================
}  // extern "C"
namespace {

#ifndef SPH_EMU
// SphTransport over the context's NCCL communicator (user = the SphCtx); ncclInt8 = 0
int nccl_group_start(void *) { return g_nccl.GroupStart(); }
int nccl_group_end(void *, void *) { return g_nccl.GroupEnd(); }
int nccl_send(void *user, const void *buf, uint64_t bytes, int32_t peer, void *stream) {
    return g_nccl.Send(buf, (size_t)bytes, 0, peer, static_cast<SphCtx *>(user)->nccl_comm, static_cast<cudaStream_t>(stream));
}
int nccl_recv(void *user, void *buf, uint64_t bytes, int32_t peer, void *stream) {
    return g_nccl.Recv(buf, (size_t)bytes, 0, peer, static_cast<SphCtx *>(user)->nccl_comm, static_cast<cudaStream_t>(stream));
}
#endif

// transport calls are host calls: under stream capture NCCL records its own kernels; the host-emulated build
// records the call itself so that a graph replay repeats it
#ifdef SPH_EMU
#define TRANSPORT_OP(st, expr) emu::submit((st), [=]() { (void)(expr); })
#else
#define TRANSPORT_OP(st, expr)                                                                                  \
    do {                                                                                                        \
        int _rc = (expr);                                                                                       \
        if (_rc) return fail(c, SPH_E_NCCL, std::string("halo exchange transport failed: ") + #expr + " -> " + std::to_string(_rc)); \
    } while (0)
#endif

// One send + recv of `bytes` with `peer` inside a transport group; counts the bytes this rank sent.
int xfer_pair(SphCtx *c, cudaStream_t st, int peer, const void *sp, void *rp, uint64_t bytes) {
    const SphTransport t = c->transport;
    TRANSPORT_OP(st, t.send(t.user, sp, bytes, peer, st));
    TRANSPORT_OP(st, t.recv(t.user, rp, bytes, peer, st));
    c->xfer_bytes += bytes;
    return SPH_OK;
}

// One-way messages inside a transport group (sph_shard_dump's gather); a send counts its bytes.
int xfer_send(SphCtx *c, cudaStream_t st, int peer, const void *sp, uint64_t bytes) {
    const SphTransport t = c->transport;
    TRANSPORT_OP(st, t.send(t.user, sp, bytes, peer, st));
    c->xfer_bytes += bytes;
    return SPH_OK;
}
int xfer_recv(SphCtx *c, cudaStream_t st, int peer, void *rp, uint64_t bytes) {
    const SphTransport t = c->transport;
    TRANSPORT_OP(st, t.recv(t.user, rp, bytes, peer, st));
    return SPH_OK;
}

// One transport group: per_side(side, peer) for each neighbour this rank has (side 0 = rank - 1, side 1 = rank + 1),
// then tail(), both issuing their messages through xfer_pair.
template <typename PerSide, typename Tail>
int transport_group(SphCtx *c, cudaStream_t st, PerSide per_side, Tail tail) {
    if (!c->has_transport) return fail(c, SPH_E_ARG, "no transport: call sph_comm_init_nccl or sph_comm_set_transport first");
    const SphTransport t = c->transport;
    TRANSPORT_OP(st, t.group_start(t.user));
    c->xfer_groups += 1;
    for (int side = 0; side < 2; ++side) {
        const int peer = side == 0 ? c->rank - 1 : c->rank + 1;
        if (peer < 0 || peer >= c->world) continue;
        if (int rc = per_side(side, peer)) return rc;
    }
    if (int rc = tail()) return rc;
    TRANSPORT_OP(st, t.group_end(t.user, st));
    return SPH_OK;
}

// One halo exchange: the packed staging of both sides goes out, the neighbours' records land behind the live
// records of the CURRENT buffer set (left neighbour's at n - 2 * halo_cap, right neighbour's at n - halo_cap),
// their headers in the device step state.  Fixed-size messages (the record count travels in the header), so the
// whole group can be captured in a CUDA graph.
int shard_exchange(SphCtx *c, cudaStream_t st, bool wide) {
    if (c->world <= 1) return SPH_OK;
    const DevArrays S = c->S;
    const uint64_t bytes = (uint64_t)(wide ? c->P.halo_cap : c->narrow_cap) * 16;
    float4 *cur[4] = {S.posm, S.veld, S.x0id, S.misc};
    return transport_group(
        c, st,
        [&](int side, int peer) {
            const int64_t tail = (int64_t)c->P.n - (side == 0 ? 2 : 1) * (int64_t)c->P.halo_cap;
            for (int k = 0; k < 4; ++k)
                if (int rc = xfer_pair(c, st, peer, S.stage[side][k], cur[k] + tail, bytes)) return rc;
            return xfer_pair(c, st, peer, S.stage_hdr[side], S.sd + (side == 0 ? SD_HDR_L : SD_HDR_R), SHARD_HDR_BYTES);
        },
        [] { return SPH_OK; });
}

// The opening of every sharded sequence: plan -> classify + sort -> info.
// wide: this sequence's exchange feeds a re-balancing step and carries sgw + 2 layers instead of sgw + 1
int shard_sort(SphCtx *c, cudaStream_t st, bool wide, int64_t *kernels) {
    k_shard_plan<<<1, 32, 0, st>>>(c->P, c->S);
    *kernels += 1;
    int rc = launch_neighbor_build(c, st, nullptr, kernels, /*move_acc=*/false);
    if (rc) return rc;
    k_shard_info<<<1, 32, 0, st>>>(c->P, c->S, c->P.sgw + (wide ? 2 : 1), wide ? c->P.halo_cap : c->narrow_cap);
    *kernels += 1;
    return SPH_OK;
}

// shard_sort -> boundary densities -> boundary forces (-> staging) ->
// { exchange || interior densities -> apply -> interior forces }
// ev[8] (optional): CUDA events at the stage boundaries, [5..6] around the exchange, [7] after the interior
// densities (sph_shard_profile_step)
int shard_sequence(SphCtx *c, cudaStream_t st, bool compute, bool wide, int64_t *kernels, cudaEvent_t *ev = nullptr) {
    if (ev) cudaEventRecord(ev[0], st);
    int rc = shard_sort(c, st, wide, kernels);
    if (rc) return rc;
    if (ev) cudaEventRecord(ev[1], st);
    const dim3 pack_grid(blocks_for(c->P.halo_cap, 256), 2);
    if (compute) {
        // boundary first: densities within one layer of the send ranges (split_density; otherwise all densities),
        // then forces + integration of the send ranges -- written into the send staging, not into the arrays: the
        // interior densities still read these positions
        launch_pair_density(c, st, kernels, /*split_mode=*/c->split_density ? 1 : 0);
        if (ev) cudaEventRecord(ev[2], st);
        launch_pair_force_and_advect(c, st, nullptr, kernels, /*split_mode=*/1);
    } else {
        if (ev) cudaEventRecord(ev[2], st);
        k_shard_apply<<<pack_grid, 256, 0, st>>>(c->P, c->S, /*copy_all=*/1);  // first exchange: the unchanged records
        *kernels += 1;
    }
    CUDA_TRY(c, cudaGetLastError());
    if (ev) cudaEventRecord(ev[3], st);
    // the exchange for the NEXT step runs on the communication stream while the interior is computed
#ifdef SPH_EMU
    cudaStream_t cs = st;  // the emulated runtime is synchronous
#else
    cudaStream_t cs = c->comm_stream;
    CUDA_TRY(c, cudaEventRecord(c->ev_packed, st));
    CUDA_TRY(c, cudaStreamWaitEvent(cs, c->ev_packed, 0));
#endif
    if (ev) cudaEventRecord(ev[5], cs);
    rc = shard_exchange(c, cs, wide);
    if (rc) return rc;
    if (ev) cudaEventRecord(ev[6], cs);
    if (compute) {
        if (c->split_density) launch_pair_density(c, st, kernels, /*split_mode=*/2);
        if (ev) cudaEventRecord(ev[7], st);
        k_shard_apply<<<pack_grid, 256, 0, st>>>(c->P, c->S, /*copy_all=*/0);  // boundary particles take their new state
        *kernels += 1;
        launch_pair_force_and_advect(c, st, nullptr, kernels, /*split_mode=*/2);
    }
#ifndef SPH_EMU
    CUDA_TRY(c, cudaEventRecord(c->ev_exchanged, cs));
    CUDA_TRY(c, cudaStreamWaitEvent(st, c->ev_exchanged, 0));
#endif
    if (ev) cudaEventRecord(ev[4], st);
    CUDA_TRY(c, cudaGetLastError());
    c->built = false; c->list_valid = false;
    return SPH_OK;
}

inline float4 *shard_body_tables(const SphCtx *c) { return reinterpret_cast<float4 *>(c->shard_buf + c->SL.off_body); }
inline int64_t body_particles(const std::vector<SphRigidBody> &bodies) {
    int64_t n = 0;
    for (const SphRigidBody &b : bodies) n += b.solid_end - b.solid_begin;
    return n;
}

// Sharded steps with dynamic solids, after the sort (and, in the Jacobi solvers' step, after the ghost alignment, which
// reorders records inside cells): the solid-id slot map of the live records, then the moving boundary volumes of the
// owned layers and ghost layers 1-2.
int launch_shard_solid_slots(SphCtx *c, cudaStream_t st, int64_t *kernels) {
    const DevParams &P = c->P;
    if (P.n_solid == 0) return SPH_OK;
    // k_rank_move also wrote the slots of trash records: only the live ones may be walked
    CUDA_TRY(c, cudaMemsetAsync(c->S.solid_slot, 0xff, (size_t)P.n_solid * 4, st));
    k_shard_solid_slots<<<step_grid(c, P.n, 256, 8), 256, 0, st>>>(P, c->S);
    *kernels += 1;
    if (c->has_dynamic_solids) {
        k_boundary_volume<true><<<blocks_for((int64_t)P.n_solid * 32, 128), 128, 0, st>>>(P, c->S, /*moving=*/1);
        *kernels += 1;
    }
    return SPH_OK;
}

// solve_rigid_body of a sharded step: k_rigid's solve on every rank from the records of all body particles, gathered in
// one transport group, then the clamps of the dynamic solids outside every body.
int launch_shard_body_solve(SphCtx *c, cudaStream_t st, int64_t *kernels) {
    const DevParams &P = c->P;
    const int nb = (int)c->bodies.size();
    if (nb == 0) return SPH_OK;
    const int64_t n_rec = body_particles(c->bodies);
    float4 *tables = shard_body_tables(c);
    float4 *mine = tables + 2 * (size_t)c->rank * n_rec;
    k_shard_body_pack<<<nb, 256, 0, st>>>(P, c->S, dev_bodies(c), mine);
    *kernels += 1;
    CUDA_TRY(c, cudaGetLastError());
    if (c->world > 1) {
        const uint64_t bytes = (uint64_t)n_rec * 32;
        int rc = transport_group(
            c, st, [](int, int) { return SPH_OK; },
            [&] {
                for (int r = 0; r < c->world; ++r) {
                    if (r == c->rank) continue;
                    if (int rc2 = xfer_pair(c, st, r, mine, tables + 2 * (size_t)r * n_rec, bytes)) return rc2;
                }
                return SPH_OK;
            });
        if (rc) return rc;
    }
    k_shard_body_solve<<<nb, RIGID_THREADS, 0, st>>>(P, c->S, dev_bodies(c), nb, tables, (int)n_rec, c->world);
    k_enforce_boundary_solid<true><<<blocks_for(P.n_solid, 256), 256, 0, st>>>(P, c->S, nb, dev_bodies(c), nb);
    *kernels += 2;
    return SPH_OK;
}

// One sharded WCSPH SPHBase.step() with dynamic solids (sph_shard_configure_bodies), in the order of launch_step +
// launch_rigid_solve, on one stream and without overlap:
//   shard_sort -> solid-id slot map -> moving boundary volumes (owned + ghost layers 1-2)
//   -> densities (owned + ghost layer 1) -> forces + integration of the owned fluid (no reaction scatter)
//   -> reactions gathered onto the owned dynamic solids + their advection -> body-particle records -> all-gather ->
//   k_rigid's solve + clamps on every rank -> clamps of the other dynamic solids -> pack the send ranges -> the record
//   exchange
int shard_bodies_sequence(SphCtx *c, cudaStream_t st, bool wide, int64_t *kernels) {
    int rc = shard_sort(c, st, wide, kernels);
    if (rc) return rc;
    const DevParams &P = c->P;
    rc = launch_shard_solid_slots(c, st, kernels);
    if (rc) return rc;
    launch_pair_density(c, st, kernels, /*split_mode=*/0);
    PDL_LAUNCH((k_force_packed<FORCE_BATCH, FORCE_THREADS, true>), blocks_for(P.n, FORCE_THREADS), FORCE_THREADS, st,
               P, c->S, 0);
    *kernels += 1;
    CUDA_TRY(c, cudaGetLastError());
    if (P.n_solid > 0) {
        k_shard_reactions<<<blocks_for((int64_t)P.n_solid * 32, 128), 128, 0, st>>>(P, c->S);
        *kernels += 1;
    }
    rc = launch_shard_body_solve(c, st, kernels);
    if (rc) return rc;
    k_shard_apply<<<dim3(blocks_for(P.halo_cap, 256), 2), 256, 0, st>>>(P, c->S, /*copy_all=*/1);
    *kernels += 1;
    CUDA_TRY(c, cudaGetLastError());
    rc = shard_exchange(c, st, wide);
    if (rc) return rc;
    c->built = false; c->list_valid = false;
    return SPH_OK;
}

}  // namespace
extern "C" {

int sph_comm_unique_id(char out128[128]) {
#ifdef SPH_EMU
    (void)out128;
    return fail(nullptr, SPH_E_NCCL, "the host-emulated build has no NCCL: use sph_comm_set_transport");
#else
    if (!out128) return SPH_E_ARG;
    if (!load_nccl()) return fail(nullptr, SPH_E_NCCL, g_nccl.err);
    NcclId id;
    int rc = g_nccl.GetUniqueId(&id);
    if (rc) return fail(nullptr, SPH_E_NCCL, std::string("ncclGetUniqueId: ") + g_nccl.GetErrorString(rc));
    std::memcpy(out128, id.internal, 128);
    return SPH_OK;
#endif
}

int sph_comm_init_nccl(SphCtx *ctx, const char id128[128], int32_t rank, int32_t world) {
    if (!ctx || !id128 || world < 1 || rank < 0 || rank >= world) return SPH_E_ARG;
#ifdef SPH_EMU
    return fail(ctx, SPH_E_NCCL, "the host-emulated build has no NCCL: use sph_comm_set_transport");
#else
    if (!load_nccl()) return fail(ctx, SPH_E_NCCL, g_nccl.err);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    NcclId id;
    std::memcpy(id.internal, id128, 128);
    int rc = g_nccl.CommInitRank(&ctx->nccl_comm, world, id, rank);
    if (rc) return fail(ctx, SPH_E_NCCL, std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(rc));
    ctx->transport = SphTransport{ctx, nccl_group_start, nccl_group_end, nccl_send, nccl_recv};
    ctx->has_transport = true;
    ctx->rank = rank; ctx->world = world;
    drop_graphs(ctx);
    return SPH_OK;
#endif
}

int sph_comm_set_transport(SphCtx *ctx, const SphTransport *t, int32_t rank, int32_t world) {
    if (!ctx || world < 1 || rank < 0 || rank >= world) return SPH_E_ARG;
    if (world > 1 && (!t || !t->group_start || !t->group_end || !t->send || !t->recv)) return fail(ctx, SPH_E_ARG, "incomplete transport");
    if (t) ctx->transport = *t;
    ctx->has_transport = t != nullptr;
    ctx->rank = rank; ctx->world = world;
    drop_graphs(ctx);
    return SPH_OK;
}

}  // extern "C"
namespace {
// The part of sph_shard_configure(_bodies) behind the argument checks: the shard buffer (n_body_particles > 0: with
// the body-particle tables), the device step state and slab mode.
int shard_setup(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                int32_t rebalance_every, int64_t n_body_particles) {
    const int32_t n_mine = ctx->P.n;
    drop_graphs(ctx);
    if (ctx->shard_buf) { cudaFree(ctx->shard_buf); ctx->shard_buf = nullptr; }
    ctx->shard = ShardMode::Off; ctx->P.slab_on = 0;
    ctx->SL = make_shard_layout(halo_capacity, ctx->world, n_body_particles);
    CUDA_TRY(ctx, cudaMalloc(reinterpret_cast<void **>(&ctx->shard_buf), ctx->SL.total));
    CUDA_TRY(ctx, cudaMemset(ctx->shard_buf, 0, ctx->SL.total));
    int32_t sd[SD_INTS] = {0};
    sd[SD_N_LIVE] = n_mine; sd[SD_OWNED] = n_mine; sd[SD_SX0] = x_lo; sd[SD_SX1] = x_hi;
    CUDA_TRY(ctx, cudaMemcpy(ctx->shard_buf + ctx->SL.off_state, sd, sizeof(sd), cudaMemcpyHostToDevice));
    ctx->shard = ShardMode::Static; ctx->P.slab_on = 1; ctx->P.sgw = ghost_layers; ctx->P.halo_cap = (int32_t)halo_capacity;
    ctx->P.has_left = ctx->rank > 0; ctx->P.has_right = ctx->rank + 1 < ctx->world;
    ctx->P.rebalance_every = rebalance_every;
    ctx->narrow_cap = (int32_t)((halo_capacity * (ghost_layers + 1) + ghost_layers + 1) / (ghost_layers + 2));
    // halo_capacity covers ghost_layers + 2 layers: the alignment carries ghost_layers of them, a sweep one
    ctx->align_cap = (int32_t)((halo_capacity * ghost_layers + ghost_layers + 1) / (ghost_layers + 2));
    ctx->sweep_cap = (int32_t)((halo_capacity + ghost_layers + 1) / (ghost_layers + 2));
    ctx->shard_world = ctx->world;
    ctx->shard_sequences = 0;
    ctx->split_density = ctx->world > 4;
    if (const char *v = std::getenv("SPH_SHARD_SPLIT_DENSITY")) ctx->split_density = std::atoi(v) != 0;
    ctx->P.n = (int32_t)ctx->n_max;  // from here on n is the CAPACITY; the live count is device state
    ctx->shard_begun = false;
    bind_arrays(ctx);
#ifndef SPH_EMU
    if (!ctx->comm_stream) {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);  // the exchange must get SMs while the interior pass runs
        CUDA_TRY(ctx, cudaStreamCreateWithPriority(&ctx->comm_stream, cudaStreamNonBlocking, hi));
        CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_packed, cudaEventDisableTiming));
        CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->ev_exchanged, cudaEventDisableTiming));
    }
#endif
    return SPH_OK;
}

// The slab arguments of both configure paths: the range (with ghost_layers >= 1, or >= 3 after it for bodies), then
// `refusal` (may be NULL: why this path does not take the context), the fluid, the capacity and rebalance_every.
int check_slab_args(SphCtx *ctx, bool bodies, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                    int32_t rebalance_every, const char *refusal) {
    if (x_lo < 0 || x_hi > ctx->P.gx || (!bodies && ghost_layers < 1) || x_hi - x_lo < ghost_layers + 2)
        return fail(ctx, SPH_E_ARG, "slab must lie inside the grid and be at least ghost_layers + 2 cell layers wide");
    if (bodies && ghost_layers < 3)
        return fail(ctx, SPH_E_ARG, "dynamic solids need ghost_layers >= 3: the moving boundary volumes of the second "
                                    "ghost layer (read by the first layer's densities) sum solids of the third");
    if (refusal) return fail(ctx, SPH_E_ARG, refusal);
    if (!ctx->P.uniform_fluid)
        return fail(ctx, SPH_E_ARG, "x-slab sharding needs a single fluid density (uniform fluid masses)");
    if (halo_capacity < 1 || 2 * halo_capacity + ctx->P.n > ctx->n_max)
        return fail(ctx, SPH_E_CAPACITY, "capacity: packed particles + 2 * halo_capacity receive slots exceed n_max");
    if (rebalance_every < 0) return SPH_E_ARG;
    return SPH_OK;
}

// sph_shard_configure_bodies (iisph = false: a WCSPH context) and sph_shard_configure_iisph_bodies (iisph = true: an
// IISPH context): the same checks and set-up, only the solver asked for differs.
int shard_configure_bodies(SphCtx *ctx, bool iisph, int32_t x_lo, int32_t x_hi, int32_t ghost_layers,
                           int64_t halo_capacity, int32_t rebalance_every, const SphRigidBody *bodies, int32_t n_bodies) {
    if (!ctx || n_bodies < 0 || (n_bodies > 0 && !bodies)) return SPH_E_ARG;
    if (ctx->solver == Solver::PCISPH) return fail(ctx, SPH_E_ARG, kPcisphSingleGpu);
    if ((ctx->solver == Solver::IISPH) != iisph)
        return fail(ctx, SPH_E_ARG, iisph ? kShardIisphBodiesContext : kShardBodiesIisph);
    if (int rc = check_slab_args(ctx, true, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every,
                                 ctx->solver == Solver::DFSPH ? kShardBodiesWcsph : nullptr))
        return rc;
    if (n_bodies > ctx->body_cap) return fail(ctx, SPH_E_CAPACITY, "more rigid bodies than the workspace was sized for");
    for (int b = 0; b < n_bodies; ++b) {
        const SphRigidBody &B = bodies[b];
        if (B.solid_begin < 0 || B.solid_end < B.solid_begin || B.solid_end > ctx->P.n_solid)
            return fail(ctx, SPH_E_ARG, "rigid body solid-id range out of bounds (pack the whole scene's solid count first)");
        for (int k = 0; k < 3; ++k)
            if (!std::isfinite(B.rest_cm[k]))
                return fail(ctx, SPH_E_ARG, "a sharded body needs its rest centre of mass (computed over the whole scene)");
    }
    // on failure the context keeps its previous body table
    const std::vector<SphRigidBody> old = ctx->bodies;
    int rc = store_bodies(ctx, bodies, n_bodies);
    if (rc == SPH_OK)
        rc = shard_setup(ctx, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every, body_particles(ctx->bodies));
    if (rc) {
        const std::string why = ctx->err;
        store_bodies(ctx, old.data(), (int32_t)old.size());
        ctx->err = why;
        return rc;
    }
    ctx->shard = ShardMode::Bodies;
    return SPH_OK;
}

// the exchange at the end of sequence q delivers the records plan kernel q + 1 works on; that one re-balances
inline bool shard_wide(const SphCtx *c) {
    const int64_t next_plan = c->shard_sequences + 1;
    return c->P.rebalance_every > 0 && next_plan % c->P.rebalance_every == 0;
}

// The sharded step entry points: their mode checks, then nsteps sequences; sequence(wide) issues one (see shard_sort)
template <typename Sequence>
int run_shard_steps(SphCtx *ctx, int32_t nsteps, const Need &need, bool args_ok, Sequence sequence) {
    if (int rc = require(ctx, need, args_ok)) return rc;
    for (int s = 0; s < nsteps; ++s) {
        if (int rc = sequence(shard_wide(ctx))) return rc;
        ctx->shard_sequences += 1;
    }
    return SPH_OK;
}
}  // namespace
extern "C" {

int sph_shard_configure(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                        int32_t rebalance_every) {
    if (!ctx) return SPH_E_ARG;
    if (ctx->solver == Solver::PCISPH) return fail(ctx, SPH_E_ARG, kPcisphSingleGpu);
    // Static solids travel in the records like fluid particles and never change; dynamic solids need moving boundary
    // volumes one ghost layer deeper, reactions across a cut and a per-body reduction across ranks: the opt-in
    // sph_shard_configure_bodies.
    const bool dynamic = !ctx->bodies.empty() || (ctx->P.n_solid > 0 && ctx->has_dynamic_solids);
    if (int rc = check_slab_args(ctx, false, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every,
                                 dynamic ? kShardStaticOnly : nullptr))
        return rc;
    return shard_setup(ctx, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every, 0);
}

int sph_shard_configure_pcisph(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                               int32_t rebalance_every) {
    if (!ctx) return SPH_E_ARG;
    if (ctx->solver != Solver::PCISPH) return fail(ctx, SPH_E_ARG, kShardPcisphContext);
    // PCISPH scatters the reactions onto dynamic solids once per step, after its loop: a reaction gather like IISPH's
    // would carry over, but it is not written
    const bool dynamic = !ctx->bodies.empty() || (ctx->P.n_solid > 0 && ctx->has_dynamic_solids);
    if (int rc = check_slab_args(ctx, false, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every,
                                 dynamic ? kShardBodiesPcisph : nullptr))
        return rc;
    return shard_setup(ctx, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every, 0);
}

int sph_shard_configure_bodies(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers, int64_t halo_capacity,
                               int32_t rebalance_every, const SphRigidBody *bodies, int32_t n_bodies) {
    return shard_configure_bodies(ctx, false, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every, bodies, n_bodies);
}

int sph_shard_configure_iisph_bodies(SphCtx *ctx, int32_t x_lo, int32_t x_hi, int32_t ghost_layers,
                                     int64_t halo_capacity, int32_t rebalance_every, const SphRigidBody *bodies,
                                     int32_t n_bodies) {
    return shard_configure_bodies(ctx, true, x_lo, x_hi, ghost_layers, halo_capacity, rebalance_every, bodies, n_bodies);
}

int sph_shard_begin(SphCtx *ctx, void *stream) {
    if (int rc = require(ctx, Need().sharded())) return rc;
    ctx->shard_sequences = 0;
    int rc = shard_sequence(ctx, static_cast<cudaStream_t>(stream), /*compute=*/false, shard_wide(ctx), &ctx->launches);
    if (rc) return rc;
    ctx->shard_sequences = 1;
    ctx->shard_begun = true;
    return SPH_OK;
}

int sph_halo_exchange(SphCtx *ctx, void *stream) {
    if (int rc = require(ctx, Need().sharded())) return rc;
    return shard_exchange(ctx, static_cast<cudaStream_t>(stream), /*wide=*/true);
}

int sph_shard_step(SphCtx *ctx, int32_t nsteps, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Need need = Need().shard_step(Solver::WCSPH, "sph_shard_step is the WCSPH step; DFSPH contexts step with "
                                                 "sph_shard_dfsph_step");
    // The world size sized the per-rank body tables of a body context; a static WCSPH context has no per-rank buffer
    // and does not check it.  Body contexts always step eagerly: SPH_SHARD_GRAPH does not apply.
    if (ctx && ctx->shard == ShardMode::Bodies)
        return run_shard_steps(
            ctx, nsteps, need.same_world("the transport's world size changed after sph_shard_configure_bodies: configure again"),
            nsteps >= 0, [&](bool wide) { return shard_bodies_sequence(ctx, st, wide, &ctx->launches); });
    // Un-graphed launches are the DEFAULT here: nothing in a sharded step waits for the host any more, so the launches
    // run ahead of the device, and a graph replay -- whose two branches (exchange || interior forces) must both finish
    // before the next replay may start -- holds back the next step's first kernels, which un-graphed launches queue
    // behind the interior pass (not measured on H100s).  SPH_SHARD_GRAPH=1 replays the captured graph instead
    // (one graph per ping-pong parity and exchange width; pays off for small per-rank problems).
    static const bool eager = !(std::getenv("SPH_SHARD_GRAPH") && std::atoi(std::getenv("SPH_SHARD_GRAPH")) != 0);
    return run_shard_steps(ctx, nsteps, need, nsteps >= 0, [&](bool wide) {
        auto issue = [&](cudaStream_t cs, int64_t *kernels) { return shard_sequence(ctx, cs, /*compute=*/true, wide, kernels); };
        // relaxed capture: NCCL may issue CUDA calls of its own while its send / recv kernels are being captured
        return eager ? issue(st, &ctx->launches)
                     : replay_graph(ctx, st, ctx->graph_shard[ctx->parity][wide], 1, cudaStreamCaptureModeRelaxed,
                                    "sharded graph", issue);
    });
}

int sph_shard_info(SphCtx *ctx, int32_t *out16, uint64_t *out_sent, void *stream) {
    if (int rc = require(ctx, Need().sharded(), out16 != nullptr)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int32_t sd[SD_INTS];
    uint32_t status = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(sd, ctx->S.sd, sizeof(sd), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(&status, ctx->S.status, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    for (int k = 0; k < 14; ++k) out16[k] = sd[k];
    out16[14] = (int32_t)status; out16[15] = 0;
    if (out_sent) *out_sent = ((uint64_t)(uint32_t)sd[SD_SENT_HI] << 32) | (uint32_t)sd[SD_SENT_LO];
    return SPH_OK;
}

// What every rank tells every other rank before the gather of sph_shard_dump (16 bytes)
struct DumpHeader {
    int64_t capacity;
    int32_t rows;
    uint32_t status;
};
static_assert(sizeof(DumpHeader) == 16, "the dump header travels as 16 bytes");

int sph_shard_dump(SphCtx *ctx, int32_t object_id, float *x, float *v, int64_t capacity, int64_t *rows_out,
                   uint32_t *status_out, void *stream) {
    if (int rc = require(ctx, Need().sharded())) return rc;
    if (!x || !v || !rows_out || !status_out || capacity < 0)
        return fail(ctx, SPH_E_ARG, "sph_shard_dump: x, v, rows_out and status_out must be non-null and capacity >= 0");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int world = ctx->world, rank = ctx->rank;
    // the owned range of the last sort sizes the grid
    int32_t own[2] = {0, 0};
    CUDA_TRY(ctx, cudaMemcpyAsync(own, ctx->S.sd + SD_OWN0, sizeof(own), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    const int n_tiles = (int)((std::max(own[1] - own[0], 0) + DUMP_TILE - 1) / DUMP_TILE);
    const uint64_t off_recv = 256, off_counts = off_recv + align_up((uint64_t)world * sizeof(DumpHeader), 256);
    const uint64_t need = off_counts + (uint64_t)(n_tiles + 1) * 4;
    if (need > ctx->dump_bytes) {
        if (ctx->dump_buf) cudaFree(ctx->dump_buf);
        ctx->dump_buf = nullptr; ctx->dump_bytes = 0;
        CUDA_TRY(ctx, cudaMalloc(reinterpret_cast<void **>(&ctx->dump_buf), need));
        ctx->dump_bytes = need;
    }
    DumpHeader *hdr_send = reinterpret_cast<DumpHeader *>(ctx->dump_buf);
    DumpHeader *hdr_recv = reinterpret_cast<DumpHeader *>(ctx->dump_buf + off_recv);
    int32_t *counts = reinterpret_cast<int32_t *>(ctx->dump_buf + off_counts);
    if (n_tiles > 0) {
        k_dump_count<<<n_tiles, DUMP_THREADS, 0, st>>>(ctx->S, own[0], own[1], object_id, counts);
        k_dump_scan<<<1, DUMP_THREADS, 0, st>>>(counts, n_tiles);
        ctx->launches += 2;
        CUDA_TRY(ctx, cudaGetLastError());
    } else {
        CUDA_TRY(ctx, cudaMemsetAsync(counts, 0, 4, st));
    }
    DumpHeader mine{capacity, 0, 0u};
    CUDA_TRY(ctx, cudaMemcpyAsync(&mine.rows, counts + n_tiles, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(&mine.status, ctx->S.status, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    // group 1: {capacity, rows, status} to every other rank, so that every rank takes the same decision below
    std::vector<DumpHeader> all((size_t)world, DumpHeader{0, 0, 0u});
    if (world > 1) {
        CUDA_TRY(ctx, cudaMemcpyAsync(hdr_send, &mine, sizeof(mine), cudaMemcpyHostToDevice, st));
        int rc = transport_group(
            ctx, st, [](int, int) { return SPH_OK; },
            [&] {
                for (int r = 0; r < world; ++r) {
                    if (r == rank) continue;
                    if (int rc2 = xfer_pair(ctx, st, r, hdr_send, hdr_recv + r, sizeof(DumpHeader))) return rc2;
                }
                return SPH_OK;
            });
        if (rc) return rc;
        CUDA_TRY(ctx, cudaMemcpyAsync(all.data(), hdr_recv, (size_t)world * sizeof(DumpHeader), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
    }
    all[(size_t)rank] = mine;
    int64_t total = 0;
    uint32_t status = 0u;
    for (const DumpHeader &h : all) { total += h.rows; status |= h.status; }
    *rows_out = rank == 0 ? total : mine.rows;
    *status_out = status;
    // the same check, in rank order, on every rank: all of them return here, or none does
    if (all[0].capacity < total)
        return fail(ctx, SPH_E_CAPACITY, "sph_shard_dump: capacity: rank 0 gathers " + std::to_string(total) + " rows of object " +
                                         std::to_string(object_id) + " but its capacity is " + std::to_string(all[0].capacity) + " rows");
    for (int r = 1; r < world; ++r)
        if (all[(size_t)r].capacity < all[(size_t)r].rows)
            return fail(ctx, SPH_E_CAPACITY, "sph_shard_dump: capacity: rank " + std::to_string(r) + " holds " +
                                             std::to_string(all[(size_t)r].rows) + " rows of object " + std::to_string(object_id) +
                                             " but its capacity is " + std::to_string(all[(size_t)r].capacity) + " rows");
    if (mine.rows > 0) {
        k_dump_scatter<<<n_tiles, DUMP_THREADS, 0, st>>>(ctx->S, own[0], own[1], object_id, counts, x, v);
        ctx->launches += 1;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    // group 2: every other rank's rows to rank 0, behind the rows of the ranks before it; zero-row transfers skipped
    bool others = false;
    for (int r = 1; r < world; ++r) others = others || all[(size_t)r].rows > 0;
    if (others) {
        int rc = transport_group(
            ctx, st, [](int, int) { return SPH_OK; },
            [&] {
                if (rank != 0) {
                    if (mine.rows == 0) return SPH_OK;
                    const uint64_t bytes = (uint64_t)mine.rows * 12;
                    if (int rc2 = xfer_send(ctx, st, 0, x, bytes)) return rc2;
                    return xfer_send(ctx, st, 0, v, bytes);
                }
                int64_t row = all[0].rows;
                for (int r = 1; r < world; ++r) {
                    const int64_t n = all[(size_t)r].rows;
                    if (n == 0) continue;
                    if (int rc2 = xfer_recv(ctx, st, r, x + 3 * row, (uint64_t)n * 12)) return rc2;
                    if (int rc2 = xfer_recv(ctx, st, r, v + 3 * row, (uint64_t)n * 12)) return rc2;
                    row += n;
                }
                return SPH_OK;
            });
        if (rc) return rc;
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return SPH_OK;
}

int sph_shard_profile_step(SphCtx *ctx, float *ms_out6, void *stream) {
    if (int rc = require(ctx, Need().shard_step(Solver::WCSPH, "sph_shard_profile_step times the WCSPH step").no_bodies(
                                  "sph_shard_profile_step times the static-solid WCSPH step, not the step of a context "
                                  "configured by sph_shard_configure_bodies"), ms_out6 != nullptr))
        return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaEvent_t ev[8];
    for (int k = 0; k < 8; ++k) CUDA_TRY(ctx, cudaEventCreate(&ev[k]));
    int rc = shard_sequence(ctx, st, /*compute=*/true, shard_wide(ctx), &ctx->launches, ev);
    if (rc) return rc;
    ctx->shard_sequences += 1;
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    cudaEventElapsedTime(&ms_out6[0], ev[0], ev[1]);  // plan + sort + info
    cudaEventElapsedTime(&ms_out6[1], ev[1], ev[2]);  // boundary densities
    cudaEventElapsedTime(&ms_out6[2], ev[2], ev[3]);  // boundary forces (-> staging)
    cudaEventElapsedTime(&ms_out6[3], ev[3], ev[7]);  // interior densities
    cudaEventElapsedTime(&ms_out6[4], ev[7], ev[4]);  // apply + interior forces + waiting for the exchange, if any
    ms_out6[5] = 0.f;
    if (ctx->world > 1) cudaEventElapsedTime(&ms_out6[5], ev[5], ev[6]);
    for (int k = 0; k < 8; ++k) cudaEventDestroy(ev[k]);
    return SPH_OK;
}

int sph_set_dfsph(SphCtx *ctx, int32_t enable) {
    if (!ctx) return SPH_E_ARG;
    set_solver(ctx, enable ? Solver::DFSPH : Solver::WCSPH);
    return SPH_OK;
}

int sph_set_iisph(SphCtx *ctx, int32_t enable) {
    if (int rc = require(ctx, Need().unsharded(enable ? kIisphAfterConfigure : nullptr))) return rc;
    if (!enable && ctx->solver != Solver::IISPH) return SPH_OK;  // not in IISPH mode: a DFSPH or WCSPH context stays
    set_solver(ctx, enable ? Solver::IISPH : Solver::WCSPH);
    return SPH_OK;
}

int sph_set_pcisph(SphCtx *ctx, int32_t enable) {
    if (int rc = require(ctx, Need().unsharded(enable ? kPcisphSingleGpu : nullptr))) return rc;
    if (!enable && ctx->solver != Solver::PCISPH) return SPH_OK;  // not in PCISPH mode: the context stays as it is
    set_solver(ctx, enable ? Solver::PCISPH : Solver::WCSPH);
    return SPH_OK;
}

}  // extern "C"
namespace {

// Sharded DFSPH blocks of the shard buffer: the DX_* ranges + alignment headers, and one fp64 error partial per rank
inline int32_t *shard_dx(const SphCtx *c) { return reinterpret_cast<int32_t *>(c->shard_buf + c->SL.off_dx); }
inline double *shard_err_parts(const SphCtx *c) { return reinterpret_cast<double *>(c->shard_buf + c->SL.off_err); }

// One exchange of the sharded DFSPH step with both neighbours: pack -> one transport group -> unpack.
//   DX_ALIGN: the ghost alignment (4 record arrays of the sgw boundary layers + a 16-byte header per side), received
//             into the receive regions behind the live records, which stay unused until the end-of-step exchange;
//   DX_VELD / DX_DFS / DX_ACC / DX_AUX / DX_MISC: one 16-byte word per particle of the outermost owned layer, received
//             into the second staging array.
// Fixed-size messages (align_cap / sweep_cap records), so both sides always agree on the byte counts.  gather_err: the
// same group also sends this rank's fp64 error partial (ctrl->err) to every other rank and receives theirs into
// shard_err_parts() -- an all-gather of 8 bytes with plain send / recv.  ctrl (may be NULL): the pack and unpack of a
// sweep behind the converged one return at once, but its transport calls are still issued, so that every rank issues
// the same sequence.  Returns at once on a context that is not sharded or has no neighbours.
int shard_dfsph_exchange(SphCtx *c, cudaStream_t st, int what, DfsphCtrl *ctrl, bool gather_err, int64_t *kernels) {
    if (c->world <= 1 || !c->P.slab_on) return SPH_OK;
    const DevArrays S = c->S;
    const DevParams &P = c->P;
    int32_t *dx = shard_dx(c);
    double *parts = shard_err_parts(c);
    const int cap = what == DX_ALIGN ? c->align_cap : c->sweep_cap;
    const uint64_t bytes = (uint64_t)cap * 16;
    const int narr = what == DX_ALIGN ? 4 : 1;
    float4 *cur[4] = {S.posm, S.veld, S.x0id, S.misc};
    float4 *rec[2][4];
    for (int side = 0; side < 2; ++side)
        for (int k = 0; k < 4; ++k)
            rec[side][k] = what == DX_ALIGN ? cur[k] + ((int64_t)P.n - (2 - side) * (int64_t)P.halo_cap) : S.stage[side][1];
    const dim3 grid(blocks_for(cap, 256), 2);
    k_dfsph_shard_pack<<<grid, 256, 0, st>>>(P, S, dx, what, ctrl);
    CUDA_TRY(c, cudaGetLastError());
    int rc = transport_group(
        c, st,
        [&](int side, int peer) {
            for (int k = 0; k < narr; ++k)
                if (int rc = xfer_pair(c, st, peer, S.stage[side][k], rec[side][k], bytes)) return rc;
            if (what != DX_ALIGN) return SPH_OK;
            return xfer_pair(c, st, peer, dx + DX_HDR_SEND + 4 * side, dx + DX_HDR_RECV + 4 * side, 16);
        },
        [&] {
            for (int r = 0; gather_err && r < c->world; ++r) {
                if (r == c->rank) continue;
                if (int rc = xfer_pair(c, st, r, &ctrl->err, parts + r, 8)) return rc;
            }
            return SPH_OK;
        });
    if (rc) return rc;
    k_dfsph_shard_unpack<<<grid, 256, 0, st>>>(P, S, dx, what, ctrl, rec[0][0], rec[0][1], rec[0][2], rec[0][3], rec[1][0],
                                               rec[1][1], rec[1][2], rec[1][3]);
    *kernels += 2;
    CUDA_TRY(c, cudaGetLastError());
    return SPH_OK;
}

// ---- solver stages ------------------------------------------------------------------------
// One launcher per stage of DFSPH, IISPH and PCISPH, shared by their ops, substeps and device-loop sweeps: it launches
// the stage over the sorted records [0, n_grid), counts its kernels into *kernels and applies the
// stage's change to the neighbour state.  Launchers never exchange: on a sharded context the substeps and sweeps issue
// the halo messages between them.  ctrl (may be NULL): a device loop's control block.  reactions: the pressure forces
// of compute_pressure_forces, which also scatter the reactions onto dynamic solids.
void solver_densities(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    launch_pair_density(c, st, kernels, /*split_mode=*/0, n_grid);
    c->list_valid = true;
}
// cohesion = false (IISPH, PCISPH): gravity + viscosity only; sigma = 0 makes the cohesion term an exact zero
void non_pressure_forces(SphCtx *c, cudaStream_t st, int64_t n_grid, bool cohesion, int64_t *kernels) {
    DevParams P = c->P;
    if (!cohesion) P.sigma = 0.0f;
    k_dfsph_non_pressure<<<blocks_for(n_grid, 128), 128, 0, st>>>(P, c->S);
    *kernels += 1;
}
void predict_velocity(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_dfsph_predict_velocity<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S);
    *kernels += 1;
}
void dfsph_factor(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_dfsph_factor<<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S);
    *kernels += 1;
}
// mode 0: density change (divergence solve), 1: density_adv (pressure solve); the same modes for dfsph_iteration
void dfsph_density_change(SphCtx *c, cudaStream_t st, int64_t n_grid, int mode, int64_t *kernels) {
    if (mode == 0) k_dfsph_density_change<0><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S);
    else k_dfsph_density_change<1><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S);
    *kernels += 1;
}
void dfsph_multiply_factor(SphCtx *c, cudaStream_t st, int64_t n_grid, float time_step, int64_t *kernels) {
    k_dfsph_multiply_factor<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S, time_step);
    *kernels += 1;
}
void dfsph_iteration(SphCtx *c, cudaStream_t st, int64_t n_grid, int mode, DfsphCtrl *ctrl, int64_t *kernels) {
    if (mode == 0) k_dfsph_iteration<0><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    else k_dfsph_iteration<1><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    *kernels += 1;
}
void dfsph_advect(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_dfsph_advect<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S);
    *kernels += 1;
    c->built = false; c->list_valid = false;  // positions moved
}
void iisph_predict(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_iisph_predict<<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S);
    *kernels += 1;
}
void iisph_pressure_accel(SphCtx *c, cudaStream_t st, int64_t n_grid, bool reactions, DfsphCtrl *ctrl,
                          int64_t *kernels) {
    if (reactions) k_iisph_pressure_accel<true><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    else k_iisph_pressure_accel<false><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    *kernels += 1;
}
void iisph_pressure_update(SphCtx *c, cudaStream_t st, int64_t n_grid, float omega, double *err, DfsphCtrl *ctrl,
                           int64_t *kernels) {
    k_iisph_pressure_update<<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, omega, err, ctrl);
    *kernels += 1;
}
void iisph_advect(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_iisph_advect<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S);
    *kernels += 1;
    c->built = false; c->list_valid = false;  // positions moved
}
void pcisph_init(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_pcisph_init<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S);
    *kernels += 1;
}
void pcisph_predict(SphCtx *c, cudaStream_t st, int64_t n_grid, DfsphCtrl *ctrl, int64_t *kernels) {
    k_pcisph_predict<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S, ctrl);
    *kernels += 1;
}
// err_part: a sharded loop's fp64 partial of the error max (NULL otherwise)
void pcisph_update_pressure(SphCtx *c, cudaStream_t st, int64_t n_grid, float delta, int32_t *err_max, double *err_part,
                            DfsphCtrl *ctrl, int64_t *kernels) {
    k_pcisph_update_pressure<<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, delta, err_max, err_part, ctrl);
    *kernels += 1;
}
void pcisph_pressure_force(SphCtx *c, cudaStream_t st, int64_t n_grid, bool reactions, DfsphCtrl *ctrl,
                           int64_t *kernels) {
    if (reactions) k_pcisph_pressure_force<true><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    else k_pcisph_pressure_force<false><<<blocks_for(n_grid, 128), 128, 0, st>>>(c->P, c->S, ctrl);
    *kernels += 1;
}
void pcisph_advect(SphCtx *c, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    k_pcisph_advect<<<blocks_for(n_grid, 256), 256, 0, st>>>(c->P, c->S);
    *kernels += 1;
    c->built = false; c->list_valid = false;  // positions moved
}

// A Jacobi loop with its loop condition on the device: sweeps are launched in batches (the first as long as the
// caller expects the loop to run -- the previous step's count is a good guess), every sweep ends with a check kernel
// that updates the DfsphCtrl in the workspace scratch block, sweeps behind the converged one return at once, and the
// host reads the control block once per batch.  sweep(ctrl) launches one sweep, check included, counts its kernels
// and returns 0 or an SPH_E_* code.
template <typename Sweep>
int device_loop(SphCtx *ctx, int32_t first_batch, DfsphCtrl *h, cudaStream_t st, Sweep sweep) {
    DfsphCtrl *ctrl = reinterpret_cast<DfsphCtrl *>(ctx->ws + ctx->L.off_scratch);
    *h = DfsphCtrl{};
    CUDA_TRY(ctx, cudaMemsetAsync(ctrl, 0, sizeof(DfsphCtrl), st));
    if (ctx->P.n == 0) return SPH_OK;
    int batch = std::max(1, std::min(first_batch, 64));
    while (!h->done) {
        for (int s = 0; s < batch; ++s)
            if (int rc = sweep(ctrl)) return rc;
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaMemcpyAsync(h, ctrl, sizeof(DfsphCtrl), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
        batch = 2;  // the guess was short: continue in pairs
    }
    return SPH_OK;
}

// The Jacobi loop of divergence_solve (mode 0, DFSPH.py:245-254) or pressure_solve (mode 1, DFSPH.py:323-331) as a
// device_loop whose sweeps end with k_dfsph_check.
// Sharded (P.slab_on): every sweep also sends the owned boundary layer's velocities after the iteration and its
// {factor, density_adv} after the density change to the neighbours' first ghost layer, and all-gathers the error
// partials for k_dfsph_check_ranked; n_fluid is then the global fluid count.
int dfsph_solve_loop(SphCtx *ctx, int mode, int32_t max_iterations, double eta, float offset, int64_t n_fluid,
                     int32_t first_batch, DfsphCtrl *h, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    const DevParams &P = ctx->P;
    const int b128 = blocks_for(n_grid, 128);
    return device_loop(ctx, first_batch, h, st, [&](DfsphCtrl *ctrl) {
        dfsph_iteration(ctx, st, n_grid, mode, ctrl, kernels);
        int rc = shard_dfsph_exchange(ctx, st, DX_VELD, ctrl, false, kernels);
        if (rc) return rc;
        if (mode == 0) k_dfsph_density_change_err<0><<<b128, 128, 0, st>>>(P, ctx->S, offset, ctrl);
        else k_dfsph_density_change_err<1><<<b128, 128, 0, st>>>(P, ctx->S, offset, ctrl);
        rc = shard_dfsph_exchange(ctx, st, DX_DFS, ctrl, true, kernels);
        if (rc) return rc;
        if (P.slab_on)
            k_dfsph_check_ranked<<<1, 1, 0, st>>>(ctrl, shard_err_parts(ctx), ctx->rank, ctx->world, (double)n_fluid, eta,
                                                  max_iterations);
        else
            k_dfsph_check<<<1, 1, 0, st>>>(ctrl, (double)n_fluid, eta, max_iterations);
        *kernels += 2;  // the density change and the check
        return SPH_OK;
    });
}

// pressure_solve of IISPH over the sorted records [0, n_grid) as a device_loop: per sweep k_iisph_pressure_accel<false>,
// k_iisph_pressure_update (error sum fused) and k_iisph_check.
// Sharded (P.slab_on): every sweep also sends the outermost owned layer's acc = {a^p, 1} after the first pass and its
// aux = {.., p / rho^2, ..} after the second to the neighbours' first ghost layer, and all-gathers the error partials
// for k_iisph_check_ranked; n_fluid is then the global fluid count.
int iisph_solve_loop(SphCtx *ctx, int32_t max_iterations, float omega, double eta, int64_t n_fluid, int32_t first_batch,
                     DfsphCtrl *h, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    return device_loop(ctx, first_batch, h, st, [&](DfsphCtrl *ctrl) {
        iisph_pressure_accel(ctx, st, n_grid, /*reactions=*/false, ctrl, kernels);
        int rc = shard_dfsph_exchange(ctx, st, DX_ACC, ctrl, false, kernels);
        if (rc) return rc;
        iisph_pressure_update(ctx, st, n_grid, omega, &ctrl->err, ctrl, kernels);
        rc = shard_dfsph_exchange(ctx, st, DX_AUX, ctrl, true, kernels);
        if (rc) return rc;
        if (ctx->P.slab_on)
            k_iisph_check_ranked<<<1, 1, 0, st>>>(ctrl, shard_err_parts(ctx), ctx->rank, ctx->world, (double)n_fluid, eta,
                                                  max_iterations);
        else
            k_iisph_check<<<1, 1, 0, st>>>(ctrl, (double)n_fluid, eta, max_iterations);
        *kernels += 1;
        return SPH_OK;
    });
}

// The prediction-correction loop of PCISPH over the sorted records [0, n_grid) as a device_loop: per sweep
// k_pcisph_predict, k_pcisph_update_pressure (error max fused), k_pcisph_pressure_force<false> and k_pcisph_check.
// Sharded (P.slab_on): every sweep also sends the outermost owned layer's dfs = {x*, m_V} after the prediction and its
// misc.y = p after the pressure update to the neighbours' first ghost layer -- the two words of a neighbour the
// pressure force reads -- and all-gathers the fp64 error partials (ctrl->err) for k_pcisph_check_ranked.
int pcisph_solve_loop(SphCtx *ctx, float delta, double eta, int32_t min_iterations, int32_t max_iterations,
                      int32_t first_batch, DfsphCtrl *h, cudaStream_t st, int64_t n_grid, int64_t *kernels) {
    const double threshold = eta * (double)ctx->P.rho0;
    const bool ranked = ctx->P.slab_on != 0;
    return device_loop(ctx, first_batch, h, st, [&](DfsphCtrl *ctrl) {
        pcisph_predict(ctx, st, n_grid, ctrl, kernels);
        int rc = shard_dfsph_exchange(ctx, st, DX_DFS, ctrl, false, kernels);
        if (rc) return rc;
        pcisph_update_pressure(ctx, st, n_grid, delta, &ctrl->err_max, ranked ? &ctrl->err : nullptr, ctrl, kernels);
        rc = shard_dfsph_exchange(ctx, st, DX_MISC, ctrl, true, kernels);
        if (rc) return rc;
        pcisph_pressure_force(ctx, st, n_grid, /*reactions=*/false, ctrl, kernels);
        if (ranked)
            k_pcisph_check_ranked<<<1, 1, 0, st>>>(ctrl, shard_err_parts(ctx), ctx->rank, ctx->world, threshold,
                                                   min_iterations, max_iterations);
        else
            k_pcisph_check<<<1, 1, 0, st>>>(ctrl, threshold, min_iterations, max_iterations);
        *kernels += 1;
        return SPH_OK;
    });
}

// The PCISPH substep (DESIGN section 11) over the sorted records [0, n_grid): densities (+ lists) -> pci_compute_deltas
// (non-pressure forces without cohesion, then p = 0, a^p = 0) -> the prediction-correction loop ->
// compute_pressure_forces (the last sweep's a^p again, now with the reactions on dynamic solids: once per step, after
// the loop) -> pci_update_time_step.  io: constants in, counts out.  Sharded (fluid and static solids), the loop's two
// exchanges per sweep are the only messages: compute_pressure_forces reads the words the last executed sweep sent, and
// there are no reactions.
int launch_pcisph_substep(SphCtx *c, cudaStream_t st, SphPcisphStep *io, int64_t n_grid, int64_t *kernels) {
    solver_densities(c, st, n_grid, kernels);
    non_pressure_forces(c, st, n_grid, /*cohesion=*/false, kernels);
    pcisph_init(c, st, n_grid, kernels);
    DfsphCtrl h{};
    int rc = pcisph_solve_loop(c, io->delta, io->eta, io->min_iterations, io->max_iterations, io->first_batch, &h, st,
                               n_grid, kernels);
    if (rc) return rc;
    io->iterations = h.iterations; io->max_err = h.last_avg; io->first_batch = std::max(1, h.sweeps);
    pcisph_pressure_force(c, st, n_grid, /*reactions=*/true, nullptr, kernels);
    pcisph_advect(c, st, n_grid, kernels);
    return SPH_OK;
}

// IISPH.substep (DESIGN section 10) over the sorted records [0, n_grid): densities (+ lists) -> non-pressure forces
// without cohesion -> predict_advection -> pressure_solve -> compute_pressure_forces (+ reactions) -> advect.  io:
// constants in, counts out.  The exchanges run only on a sharded context: v* after predict_velocity (read by
// k_iisph_predict), aux after k_iisph_predict (the warm-start p / rho^2 the first sweep reads), then the two of every
// sweep.  compute_pressure_forces reads the aux words the converged sweep sent; nothing reads a ghost value after it.
// Sharded with dynamic solids (ShardMode::Bodies): compute_pressure_forces runs without its reaction scatter (it would add
// the reactions a second time, and onto ghost copies), the first ghost layer's final pressures arrive in one more
// message (DX_MISC) and k_iisph_shard_reactions gathers the reactions onto the owned dynamic solids before the advect.
int launch_iisph_substep(SphCtx *c, cudaStream_t st, SphIisphStep *io, int64_t n_grid, int64_t *kernels) {
    const DevParams &P = c->P;
    solver_densities(c, st, n_grid, kernels);
    non_pressure_forces(c, st, n_grid, /*cohesion=*/false, kernels);
    predict_velocity(c, st, n_grid, kernels);
    int rc = shard_dfsph_exchange(c, st, DX_VELD, nullptr, false, kernels);
    if (rc) return rc;
    iisph_predict(c, st, n_grid, kernels);
    rc = shard_dfsph_exchange(c, st, DX_AUX, nullptr, false, kernels);
    if (rc) return rc;
    DfsphCtrl h{};
    rc = iisph_solve_loop(c, io->max_iterations, io->omega, io->eta, io->n_fluid, io->first_batch, &h, st, n_grid,
                          kernels);
    if (rc) return rc;
    io->iterations = h.iterations; io->avg_err = h.last_avg; io->first_batch = std::max(1, h.sweeps);
    const bool bodies = c->shard == ShardMode::Bodies;
    iisph_pressure_accel(c, st, n_grid, /*reactions=*/!bodies, nullptr, kernels);
    if (bodies) {
        rc = shard_dfsph_exchange(c, st, DX_MISC, nullptr, false, kernels);
        if (rc) return rc;
        if (P.n_solid > 0) {
            k_iisph_shard_reactions<<<blocks_for((int64_t)P.n_solid * 32, 128), 128, 0, st>>>(P, c->S);
            *kernels += 1;
        }
    }
    iisph_advect(c, st, n_grid, kernels);
    return SPH_OK;
}

// DFSPH.substep (DFSPH.py:399-408) over the sorted records [0, n_grid), with io's constants in and its counts out:
//   densities -> factor -> [density change -> * 1/dt -> dfs exchange -> divergence loop -> * dt] -> non-pressure
//   forces -> predict velocity -> veld exchange -> density_adv -> * 1/dt^2 -> dfs exchange -> pressure loop -> advect
// The exchanges run only on a sharded context.  After its ghost alignment a ghost record holds exactly what its owner
// holds in the same position, so a value that changes on the owner is sent once per change -- veld after each Jacobi
// iteration and after predict_velocity, dfs after each density change -- and every pass reads current ghost values.
// The {factor, density_adv} words are sent AFTER the multiply_time_step that follows each loop's opening density
// change: one message carries both, and the scale at the end of the divergence loop needs no message because nothing
// reads a ghost's factor before the pressure loop's opening exchange.
int launch_dfsph_substep(SphCtx *c, cudaStream_t st, SphDfsphStep *io, int64_t n_grid, int64_t *kernels) {
    solver_densities(c, st, n_grid, kernels);
    dfsph_factor(c, st, n_grid, kernels);
    DfsphCtrl h{};
    if (io->enable_divergence_solver) {  // divergence_solve, DFSPH.py:236-276
        dfsph_density_change(c, st, n_grid, 0, kernels);
        dfsph_multiply_factor(c, st, n_grid, io->inv_dt, kernels);
        int rc = shard_dfsph_exchange(c, st, DX_DFS, nullptr, false, kernels);
        if (rc) return rc;
        rc = dfsph_solve_loop(c, 0, io->max_iterations_v, io->eta_v, 0.0f, io->n_fluid, io->first_batch_v, &h, st, n_grid,
                              kernels);
        if (rc) return rc;
        io->iterations_v = h.iterations; io->avg_err_v = h.last_avg; io->first_batch_v = std::max(1, h.sweeps);
        dfsph_multiply_factor(c, st, n_grid, io->dt, kernels);
    }
    non_pressure_forces(c, st, n_grid, /*cohesion=*/true, kernels);
    predict_velocity(c, st, n_grid, kernels);
    int rc = shard_dfsph_exchange(c, st, DX_VELD, nullptr, false, kernels);
    if (rc) return rc;
    // pressure_solve, DFSPH.py:314-352
    dfsph_density_change(c, st, n_grid, 1, kernels);
    dfsph_multiply_factor(c, st, n_grid, io->inv_dt2, kernels);
    rc = shard_dfsph_exchange(c, st, DX_DFS, nullptr, false, kernels);
    if (rc) return rc;
    rc = dfsph_solve_loop(c, 1, io->max_iterations, io->eta, io->density0, io->n_fluid, io->first_batch, &h, st, n_grid,
                          kernels);
    if (rc) return rc;
    io->iterations = h.iterations; io->avg_err = h.last_avg; io->first_batch = std::max(1, h.sweeps);
    dfsph_advect(c, st, n_grid, kernels);
    return SPH_OK;
}

// The single-GPU step entry points of the solvers whose substep launches itself (DFSPH, IISPH, PCISPH): their mode
// checks, then nsteps of SPHBase.step() (sph_base.py:263-271):
//   neighbour build -> moving boundary volumes -> substep() -> solve_rigid_body -> enforce_boundary_3D(fluid)
template <typename Substep>
int run_single_steps(SphCtx *ctx, cudaStream_t st, int32_t nsteps, const Need &need, bool args_ok, Substep substep) {
    if (int rc = require(ctx, need, args_ok)) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    for (int s = 0; s < nsteps; ++s) {
        // ps.initialize_particle_system(), compute_moving_boundary_volume() (sph_base.py:264-265)
        int rc = launch_neighbor_build(ctx, st, nullptr, &ctx->launches, /*move_acc=*/true);
        if (rc) return rc;
        if (ctx->has_dynamic_solids) { rc = launch_boundary_volume(ctx, 1, st, &ctx->launches); if (rc) return rc; }
        rc = substep();
        if (rc) return rc;
        // solve_rigid_body(), enforce_boundary_3D(fluid) (sph_base.py:270-271)
        if (!ctx->bodies.empty()) { rc = launch_rigid_solve(ctx, st, &ctx->launches); if (rc) return rc; }
        k_enforce_boundary<<<blocks_for(ctx->P.n, 256), 256, 0, st>>>(ctx->P, ctx->S, /*particle_type=*/1);
        ctx->launches += 1;
        CUDA_TRY(ctx, cudaGetLastError());
    }
    return SPH_OK;
}

// One sharded SPHBase.step() of a solver whose substep launches itself (DFSPH, IISPH, PCISPH; no overlap of the exchanges with
// computation):
//   shard_sort -> DX ranges -> ghost alignment [-> solid-id slot map -> moving boundary volumes]
//   -> substep(n_grid) on owned records + ghosts [-> body all-gather + solve -> clamps of the other dynamic solids]
//   -> clamp (owned fluid) -> pack the send ranges -> the record exchange that feeds the next step's classification
// [..]: body contexts only (ShardMode::Bodies; IISPH, sph_shard_configure_iisph_bodies).
template <typename Substep>
int shard_dfsph_sequence(SphCtx *c, cudaStream_t st, bool wide, int64_t *kernels, Substep substep) {
    const bool bodies = c->shard == ShardMode::Bodies;
    int rc = shard_sort(c, st, wide, kernels);
    if (rc) return rc;
    const DevParams &P = c->P;
    k_dfsph_shard_ranges<<<1, 32, 0, st>>>(P, c->S, shard_dx(c), c->align_cap, c->sweep_cap);
    *kernels += 1;
    CUDA_TRY(c, cudaGetLastError());
    rc = shard_dfsph_exchange(c, st, DX_ALIGN, nullptr, false, kernels);
    if (rc) return rc;
    if (bodies) { rc = launch_shard_solid_slots(c, st, kernels); if (rc) return rc; }
    // The step waits on the host once per batch of sweeps anyway; one more short wait here for the live count lets
    // every substep launch cover [0, n_live) -- owned records and ghosts -- instead of the whole capacity.
    int32_t n_live = 0;
    CUDA_TRY(c, cudaMemcpyAsync(&n_live, c->S.sd + SD_N_LIVE, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(c, cudaStreamSynchronize(st));
    const int64_t n_grid = std::min<int64_t>(std::max<int32_t>(n_live, 1), P.n);
    rc = substep(n_grid);
    if (rc) return rc;
    // solve_rigid_body(), enforce_boundary_3D(fluid) (sph_base.py:270-271)
    if (bodies) { rc = launch_shard_body_solve(c, st, kernels); if (rc) return rc; }
    k_enforce_boundary<<<blocks_for(n_grid, 256), 256, 0, st>>>(P, c->S, /*particle_type=*/1);
    // the advanced records of the send ranges -> staging, then the exchange the next step classifies
    k_shard_apply<<<dim3(blocks_for(P.halo_cap, 256), 2), 256, 0, st>>>(P, c->S, /*copy_all=*/1);
    *kernels += 2;
    CUDA_TRY(c, cudaGetLastError());
    return shard_exchange(c, st, wide);
}

}  // namespace
extern "C" {

int sph_dfsph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::DFSPH, kNoDfsph))) return rc;
    const int64_t n = ctx->P.n;
    if (n == 0) return SPH_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (op >= DFSPH_COMPUTE_DENSITIES && op <= DFSPH_NON_PRESSURE_FORCES && op != DFSPH_DENSITY_ERROR &&
        op != DFSPH_MULTIPLY_FACTOR) {
        if (!ctx->built)
            return fail(ctx, SPH_E_ARG, "neighbour structure is stale: call sph_neighbor_build first");
        if (op != DFSPH_COMPUTE_DENSITIES && !ctx->list_valid)
            return fail(ctx, SPH_E_ARG, "neighbour lists are stale: run op 0 (compute_densities) first");
    }
    int64_t *k = &ctx->launches;
    switch (op) {
        case DFSPH_COMPUTE_DENSITIES: solver_densities(ctx, st, n, k); break;
        case DFSPH_COMPUTE_FACTOR: dfsph_factor(ctx, st, n, k); break;
        case DFSPH_DENSITY_CHANGE: dfsph_density_change(ctx, st, n, 0, k); break;
        case DFSPH_DENSITY_ADV: dfsph_density_change(ctx, st, n, 1, k); break;
        case DFSPH_DENSITY_ERROR:  // the host loop's error read-back; the device loop fuses it into the density change
            if (!out_dev) return SPH_E_ARG;
            k_dfsph_density_error<<<blocks_for(n, 256), 256, 0, st>>>(ctx->P, ctx->S, arg, static_cast<double *>(out_dev));
            *k += 1;
            break;
        case DFSPH_MULTIPLY_FACTOR: dfsph_multiply_factor(ctx, st, n, arg, k); break;
        case DFSPH_DIVERGENCE_ITERATION: dfsph_iteration(ctx, st, n, 0, nullptr, k); break;
        case DFSPH_PRESSURE_ITERATION: dfsph_iteration(ctx, st, n, 1, nullptr, k); break;
        case DFSPH_NON_PRESSURE_FORCES: non_pressure_forces(ctx, st, n, /*cohesion=*/true, k); break;
        case DFSPH_PREDICT_VELOCITY: predict_velocity(ctx, st, n, k); break;
        case DFSPH_ADVECT: dfsph_advect(ctx, st, n, k); break;
        default: return fail(ctx, SPH_E_ARG, "unknown DFSPH op");
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_dfsph_solve(SphCtx *ctx, int32_t mode, int32_t max_iterations, double eta, float offset, int64_t n_fluid,
                    int32_t first_batch, int32_t *iterations_out, int32_t *sweeps_out, double *avg_err_out, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::DFSPH, kNoDfsph).fresh_lists(), (mode == 0 || mode == 1) && n_fluid >= 1))
        return rc;
    DfsphCtrl h{};
    int rc = dfsph_solve_loop(ctx, mode, max_iterations, eta, offset, n_fluid, first_batch, &h,
                              static_cast<cudaStream_t>(stream), ctx->P.n, &ctx->launches);
    if (rc) return rc;
    if (iterations_out) *iterations_out = h.iterations;
    if (sweeps_out) *sweeps_out = h.sweeps;
    if (avg_err_out) *avg_err_out = h.last_avg;
    return SPH_OK;
}

int sph_dfsph_step(SphCtx *ctx, int32_t nsteps, SphDfsphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const char *sharded = "this context is sharded: step it with sph_shard_dfsph_step";
    return run_single_steps(ctx, st, nsteps, Need().runs(Solver::DFSPH, kNoDfsph).unsharded(sharded),
                            io && nsteps >= 0 && io->n_fluid >= 1,
                            [&] { return launch_dfsph_substep(ctx, st, io, ctx->P.n, &ctx->launches); });
}

int sph_iisph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::IISPH, kNoIisph).unsharded(kIisphSharded))) return rc;
    const int64_t n = ctx->P.n;
    if (n == 0) return SPH_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (op < IISPH_COMPUTE_DENSITIES || op > IISPH_ADVECT) return fail(ctx, SPH_E_ARG, "unknown IISPH op");
    if (!ctx->built) return fail(ctx, SPH_E_ARG, "neighbour structure is stale: call sph_neighbor_build first");
    if (op != IISPH_COMPUTE_DENSITIES && op != IISPH_ADVECT && !ctx->list_valid)
        return fail(ctx, SPH_E_ARG, "neighbour lists are stale: run op 0 (compute_densities) first");
    if (op == IISPH_PRESSURE_SOLVE_ITERATION && !out_dev) return SPH_E_ARG;
    int64_t *k = &ctx->launches;
    switch (op) {
        case IISPH_COMPUTE_DENSITIES: solver_densities(ctx, st, n, k); break;
        case IISPH_NON_PRESSURE_FORCES: non_pressure_forces(ctx, st, n, /*cohesion=*/false, k); break;
        case IISPH_PREDICT_ADVECTION:
            predict_velocity(ctx, st, n, k);
            iisph_predict(ctx, st, n, k);
            break;
        case IISPH_PRESSURE_SOLVE_ITERATION:  // one sweep of iisph_solve_loop without its check
            iisph_pressure_accel(ctx, st, n, /*reactions=*/false, nullptr, k);
            iisph_pressure_update(ctx, st, n, arg, static_cast<double *>(out_dev), nullptr, k);
            break;
        case IISPH_PRESSURE_FORCES: iisph_pressure_accel(ctx, st, n, /*reactions=*/true, nullptr, k); break;
        case IISPH_ADVECT: iisph_advect(ctx, st, n, k); break;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_iisph_solve(SphCtx *ctx, int32_t max_iterations, float omega, double eta, int64_t n_fluid, int32_t first_batch,
                    int32_t *iterations_out, double *avg_err_out, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::IISPH, kNoIisph).unsharded(kIisphSharded).fresh_lists(),
                         n_fluid >= 1 && max_iterations >= 1))
        return rc;
    DfsphCtrl h{};
    int rc = iisph_solve_loop(ctx, max_iterations, omega, eta, n_fluid, first_batch, &h, static_cast<cudaStream_t>(stream),
                              ctx->P.n, &ctx->launches);
    if (rc) return rc;
    if (iterations_out) *iterations_out = h.iterations;
    if (avg_err_out) *avg_err_out = h.last_avg;
    return SPH_OK;
}

int sph_iisph_step(SphCtx *ctx, int32_t nsteps, SphIisphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_single_steps(ctx, st, nsteps, Need().runs(Solver::IISPH, kNoIisph).unsharded(kIisphSharded),
                            io && nsteps >= 0 && io->n_fluid >= 1 && io->max_iterations >= 1,
                            [&] { return launch_iisph_substep(ctx, st, io, ctx->P.n, &ctx->launches); });
}

int sph_iisph_read(SphCtx *ctx, float *a_ii, float *s, float *ap, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::IISPH, kNoIisph))) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    k_iisph_read<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, a_ii, s, ap);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_pcisph_op(SphCtx *ctx, int32_t op, float arg, void *out_dev, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::PCISPH, kNoPcisph).unsharded(kPcisphSharded))) return rc;
    const int64_t n = ctx->P.n;
    if (n == 0) return SPH_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (op < PCISPH_COMPUTE_DENSITIES || op > PCISPH_UPDATE_TIME_STEP) return fail(ctx, SPH_E_ARG, "unknown PCISPH op");
    if (!ctx->built) return fail(ctx, SPH_E_ARG, "neighbour structure is stale: call sph_neighbor_build first");
    if (op != PCISPH_COMPUTE_DENSITIES && op != PCISPH_UPDATE_TIME_STEP && !ctx->list_valid)
        return fail(ctx, SPH_E_ARG, "neighbour lists are stale: run op 0 (compute_densities) first");
    if (op == PCISPH_UPDATE_PRESSURE && !out_dev) return SPH_E_ARG;
    int64_t *k = &ctx->launches;
    switch (op) {
        case PCISPH_COMPUTE_DENSITIES: solver_densities(ctx, st, n, k); break;
        case PCISPH_COMPUTE_DELTAS:
            non_pressure_forces(ctx, st, n, /*cohesion=*/false, k);
            pcisph_init(ctx, st, n, k);
            break;
        case PCISPH_POS_VEL_PREDICTION: pcisph_predict(ctx, st, n, nullptr, k); break;
        case PCISPH_UPDATE_PRESSURE:
            pcisph_update_pressure(ctx, st, n, arg, static_cast<int32_t *>(out_dev), nullptr, nullptr, k);
            break;
        case PCISPH_UPDATE_PRESSURE_FORCE: pcisph_pressure_force(ctx, st, n, /*reactions=*/false, nullptr, k); break;
        case PCISPH_COMPUTE_PRESSURE_FORCES: pcisph_pressure_force(ctx, st, n, /*reactions=*/true, nullptr, k); break;
        case PCISPH_UPDATE_TIME_STEP: pcisph_advect(ctx, st, n, k); break;
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_pcisph_solve(SphCtx *ctx, float delta, double eta, int32_t min_iterations, int32_t max_iterations,
                     int32_t first_batch, int32_t *iterations_out, double *max_err_out, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::PCISPH, kNoPcisph).unsharded(kPcisphSharded).fresh_lists(),
                         max_iterations >= 1))
        return rc;
    DfsphCtrl h{};
    int rc = pcisph_solve_loop(ctx, delta, eta, min_iterations, max_iterations, first_batch, &h,
                               static_cast<cudaStream_t>(stream), ctx->P.n, &ctx->launches);
    if (rc) return rc;
    if (iterations_out) *iterations_out = h.iterations;
    if (max_err_out) *max_err_out = h.last_avg;
    return SPH_OK;
}

int sph_pcisph_step(SphCtx *ctx, int32_t nsteps, SphPcisphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_single_steps(ctx, st, nsteps, Need().runs(Solver::PCISPH, kNoPcisph).unsharded(kPcisphSharded),
                            io && nsteps >= 0 && io->max_iterations >= 1,
                            [&] { return launch_pcisph_substep(ctx, st, io, ctx->P.n, &ctx->launches); });
}

int sph_pcisph_read(SphCtx *ctx, float *rho_star, float *p, float *ap, void *stream) {
    if (int rc = require(ctx, Need().runs(Solver::PCISPH, kNoPcisph))) return rc;
    if (ctx->P.n == 0) return SPH_OK;
    k_pcisph_read<<<blocks_for(ctx->P.n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx->P, ctx->S, rho_star, p,
                                                                                              ap);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int sph_shard_dfsph_step(SphCtx *ctx, int32_t nsteps, SphDfsphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const char *wcsph = "sph_set_dfsph(1) was not called: WCSPH contexts step with sph_shard_step";
    Need need = Need().shard_step(Solver::DFSPH, wcsph).no_bodies(kShardBodiesWcsph).same_world(kWorldChanged);
    return run_shard_steps(ctx, nsteps, need, io && nsteps >= 0 && io->n_fluid >= 1, [&](bool wide) {
        return shard_dfsph_sequence(ctx, st, wide, &ctx->launches,
                                    [&](int64_t n_grid) { return launch_dfsph_substep(ctx, st, io, n_grid, &ctx->launches); });
    });
}

int sph_shard_iisph_step(SphCtx *ctx, int32_t nsteps, SphIisphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Need need = Need().shard_step(Solver::IISPH, "sph_set_iisph(1) was not called before sph_shard_configure");
    return run_shard_steps(ctx, nsteps, need.same_world(kWorldChanged),
                           io && nsteps >= 0 && io->n_fluid >= 1 && io->max_iterations >= 1, [&](bool wide) {
        return shard_dfsph_sequence(ctx, st, wide, &ctx->launches,
                                    [&](int64_t n_grid) { return launch_iisph_substep(ctx, st, io, n_grid, &ctx->launches); });
    });
}

int sph_shard_pcisph_step(SphCtx *ctx, int32_t nsteps, SphPcisphStep *io, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Need need = Need().shard_step(Solver::PCISPH, "sph_set_pcisph(1) was not called before sph_shard_configure_pcisph");
    return run_shard_steps(ctx, nsteps, need.same_world(kWorldChanged), io && nsteps >= 0 && io->max_iterations >= 1,
                           [&](bool wide) {
        return shard_dfsph_sequence(ctx, st, wide, &ctx->launches,
                                    [&](int64_t n_grid) { return launch_pcisph_substep(ctx, st, io, n_grid, &ctx->launches); });
    });
}

int sph_shard_transport_stats(SphCtx *ctx, uint64_t *out2) {
    if (!ctx || !out2) return SPH_E_ARG;
    out2[0] = ctx->xfer_groups;
    out2[1] = ctx->xfer_bytes;
    return SPH_OK;
}

int sph_read_status(SphCtx *ctx, uint32_t *status_out, void *stream) {
    if (!ctx || !status_out) return SPH_E_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(ctx, cudaMemcpyAsync(status_out, ctx->S.status, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    return SPH_OK;
}

int sph_clear_status(SphCtx *ctx, void *stream) {
    if (!ctx) return SPH_E_ARG;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->S.status, 0, 4, static_cast<cudaStream_t>(stream)));
    return SPH_OK;
}

int sph_neighbor_stats(SphCtx *ctx, int32_t *out_dev4, void *stream) {
    if (!ctx || !out_dev4) return SPH_E_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(ctx, cudaMemsetAsync(out_dev4, 0, 16, st));
    if (ctx->P.n == 0) return SPH_OK;
    k_neighbor_stats<<<blocks_for(ctx->P.n, 256), 256, 0, st>>>(ctx->P, ctx->S, out_dev4);
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return SPH_OK;
}

int64_t sph_particle_count(const SphCtx *ctx) { return ctx ? ctx->P.n : 0; }
int64_t sph_launch_count(const SphCtx *ctx) { return ctx ? ctx->launches : 0; }

int sph_profile_step(SphCtx *ctx, float *ms, int32_t n, void *stream) {
    if (!ctx || !ms || n <= 0) return SPH_E_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StageTimer tm;
    tm.on = true;
    tm.st = st;
    int rc = launch_step(ctx, st, &tm, &ctx->launches);
    if (rc) return rc;
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    float out[NUM_TIMERS];
    for (int k = 0; k < NUM_TIMERS; ++k) out[k] = 0.f;
    for (int k = 0; k + 1 < tm.count; ++k) {
        float t = 0.f;
        cudaEventElapsedTime(&t, tm.ev[k], tm.ev[k + 1]);
        out[tm.stage_of[k]] += t;
    }
    if (tm.count >= 2) cudaEventElapsedTime(&out[T_TOTAL], tm.ev[0], tm.ev[tm.count - 1]);
    for (int k = 0; k < tm.count; ++k) cudaEventDestroy(tm.ev[k]);
    int m = n < NUM_TIMERS ? n : NUM_TIMERS;
    for (int k = 0; k < m; ++k) ms[k] = out[k];
    return m;
}

const char *sph_timer_name(int32_t i) { return (i >= 0 && i < NUM_TIMERS) ? kTimerNames[i] : ""; }

}  // extern "C"
