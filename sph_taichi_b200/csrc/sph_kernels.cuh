// sph_kernels.cuh -- device kernels of libsph_b200 (sm_90a).  See sph_common.cuh for layout.
#pragma once
#include "sph_common.cuh"

// =====================================================================================
// state transfer (ParticleSystem fields <-> packed SoA)
// =====================================================================================
__global__ void k_pack(DevParams P, DevArrays S, SphFields F) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float m_V = F.m_V[i];
    S.posm[i] = make_float4(F.x[3 * i], F.x[3 * i + 1], F.x[3 * i + 2], m_V);
    S.veld[i] = make_float4(F.v[3 * i], F.v[3 * i + 1], F.v[3 * i + 2], F.density[i]);
    S.x0id[i] = make_float4(F.x_0[3 * i], F.x_0[3 * i + 1], F.x_0[3 * i + 2], __int_as_float(F.object_id[i]));
    uint32_t flags = (F.material[i] == SPH_MATERIAL_FLUID ? FLAG_FLUID : 0u) | (F.is_dynamic[i] ? FLAG_DYNAMIC : 0u) |
                     ((uint32_t)(F.color[3 * i] & 255) << 8) | ((uint32_t)(F.color[3 * i + 1] & 255) << 16) |
                     ((uint32_t)(F.color[3 * i + 2] & 255) << 24);
    int sid = F.solid_id ? F.solid_id[i] : -1;
    S.misc[i] = make_float4(F.m[i], F.pressure[i], __uint_as_float(flags), __int_as_float(sid));
    S.acc[i] = make_float4(F.acceleration[3 * i], F.acceleration[3 * i + 1], F.acceleration[3 * i + 2], 0.0f);
    S.aux[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    S.grid_ids[i] = 0;
    if (sid >= 0) S.solid_slot[sid] = i;
}

__global__ void k_unpack(DevParams P, DevArrays S, SphFields F) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float4 a = S.posm[i], b = S.veld[i], c = S.x0id[i], d = S.misc[i], e = S.acc[i];
    F.x[3 * i] = a.x; F.x[3 * i + 1] = a.y; F.x[3 * i + 2] = a.z; F.m_V[i] = a.w;
    F.v[3 * i] = b.x; F.v[3 * i + 1] = b.y; F.v[3 * i + 2] = b.z; F.density[i] = b.w;
    F.x_0[3 * i] = c.x; F.x_0[3 * i + 1] = c.y; F.x_0[3 * i + 2] = c.z; F.object_id[i] = __float_as_int(c.w);
    uint32_t flags = __float_as_uint(d.z);
    F.m[i] = d.x; F.pressure[i] = d.y;
    F.material[i] = (flags & FLAG_FLUID) ? SPH_MATERIAL_FLUID : SPH_MATERIAL_SOLID;
    F.is_dynamic[i] = (flags & FLAG_DYNAMIC) ? 1 : 0;
    F.color[3 * i] = (flags >> 8) & 255; F.color[3 * i + 1] = (flags >> 16) & 255; F.color[3 * i + 2] = (flags >> 24) & 255;
    F.acceleration[3 * i] = e.x; F.acceleration[3 * i + 1] = e.y; F.acceleration[3 * i + 2] = e.z;
    if (F.grid_ids) F.grid_ids[i] = S.grid_ids[i];
    if (F.solid_id) F.solid_id[i] = __float_as_int(d.w);
    if (F.dfsph_factor) F.dfsph_factor[i] = S.dfs[i].x;
    if (F.density_adv) F.density_adv[i] = S.dfs[i].y;
}

__global__ void k_unpack_xv(DevParams P, DevArrays S, float *x, float *v, int32_t *object_id) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float4 a = S.posm[i], b = S.veld[i];
    x[3 * i] = a.x; x[3 * i + 1] = a.y; x[3 * i + 2] = a.z;
    v[3 * i] = b.x; v[3 * i + 1] = b.y; v[3 * i + 2] = b.z;
    if (object_id) object_id[i] = __float_as_int(S.x0id[i].w);
}

__global__ void k_upload_xv(DevParams P, DevArrays S, const float *x, const float *v) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float4 a = S.posm[i], b = S.veld[i];
    S.posm[i] = make_float4(x[3 * i], x[3 * i + 1], x[3 * i + 2], a.w);
    S.veld[i] = make_float4(v[3 * i], v[3 * i + 1], v[3 * i + 2], b.w);
}

// =====================================================================================
// neighbour build: hash + histogram -> single-pass scan -> bucket -> stable rank + move
// (particle_system.py:311-375)
// =====================================================================================
__global__ void k_hash_count(DevParams P, DevArrays S) {
    pdl_wait();
    // sharded: the inputs are the live records of the last sort and what the halo exchange delivered (compact
    // numbering, grid-stride loop: the grid of a graph-replayed step is fixed, the counts are device state)
    const int total = P.slab_on ? shard_input_total(S.sd) : P.n;
    for (int u0 = blockIdx.x * blockDim.x; u0 < total; u0 += gridDim.x * blockDim.x) {
    const int u = u0 + threadIdx.x;
    const bool active = u < total;
    const int i = (P.slab_on && active) ? shard_input_index(P, S.sd, u) : u;
    int c = -1;
    if (active) {
        float4 p = S.posm[i];
        int ci, cj, ck;
        cell_of(P, p.x, p.y, p.z, ci, cj, ck);
        bool bad = ci < 0 || ci >= P.gx || cj < 0 || cj >= P.gy || ck < 0 || ck >= P.gz || !(p.x == p.x) ||
                   !(p.y == p.y) || !(p.z == p.z);
        if (bad) {
            // the reference writes out of bounds here; we flag it and park the particle in range
            atomicOr(S.status, SPH_STATUS_OUT_OF_GRID);
            ci = min(max(ci, 0), P.gx - 1); cj = min(max(cj, 0), P.gy - 1); ck = min(max(ck, 0), P.gz - 1);
        }
        c = (ci * P.gy + cj) * P.gz + ck;
        if (P.slab_on) {
            // Ownership is a pure function of the (bitwise identical) position on both ranks, so a
            // particle is owned by exactly one rank.  Everything that is neither owned nor inside
            // the ghost band goes to the trash bucket C, which sorts to the end.
            const int sx0 = S.sd[SD_SX0], sx1 = S.sd[SD_SX1];
            float4 m = S.misc[i];
            uint32_t fl = __float_as_uint(m.z);
            bool in_slab = ci >= sx0 && ci < sx1;
            bool in_band = ci >= sx0 - P.sgw && ci < sx1 + P.sgw;
            bool was_ghost = (fl & FLAG_GHOST) != 0;
            if (was_ghost) {
                c = P.C;  // last step's ghosts: dropped (the neighbour sends fresh copies every step)
            } else if (in_slab) {
                // stays / becomes owned
            } else if (in_band) {
                // a neighbour's particle, or one of mine that just left the slab (the neighbour adopts
                // it from the records I sent; I keep my copy as this step's ghost)
                reinterpret_cast<float *>(S.misc + i)[2] = __uint_as_float(fl | FLAG_GHOST);
            } else {
                c = P.C;  // outside the band
            }
        }
        S.cid[i] = c;
    }
    // The histogram atomic also hands out the arrival ticket inside the cell, which k_bucket turns into a slot
    // after the scan -- no second round of atomics.  The input is the previous step's sorted order, so the lanes of
    // a warp hold 4-5 distinct cells (and the trash bucket of a sharded step ~10 % of all records): ONE atomic per
    // distinct cell and warp (MATCH.ANY), the lanes of a group take consecutive tickets.  Any ticket order is
    // fine -- k_rank_move restores the stable order.
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(0xffffffffu, c);  // inactive lanes (c == -1) form their own group
    const int leader = __ffs(peers) - 1;
    int base = 0;
    if (active && lane == leader) base = atomicAdd(S.cell_end + c, __popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (active) S.ticket[i] = base + __popc(peers & ((1u << lane) - 1u));
    }
}

// ---- x-slab sharding: the per-step bookkeeping that used to live on the host (round 1: an all-gather of the
// info rows, a D2H copy and a host wait every step) -- three one-warp kernels inside the step graph ----

// Before the classification: take the record counts out of the headers the halo exchange delivered and, every
// `rebalance_every` steps, move the slab cuts by one layer toward the heavier side.  Both ranks of a cut hold
// the same four integers (their own and the neighbour's owned count and width, exchanged in the headers) and
// evaluate the same integer expression, so they always agree -- no extra message.
__device__ __forceinline__ int shard_cut_move(long long owned_l, int width_l, long long owned_r, int width_r) {
    // the cut moves one layer toward the heavier side when the difference exceeds ~1.2 layers' worth
    if ((owned_l - owned_r) * 5 * width_l > 6 * owned_l && width_l > SHARD_MIN_WIDTH) return -1;
    if ((owned_r - owned_l) * 5 * width_r > 6 * owned_r && width_r > SHARD_MIN_WIDTH) return +1;
    return 0;
}
__global__ void k_shard_plan(DevParams P, DevArrays S) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int32_t *sd = S.sd;
    const int32_t *hl = sd + SD_HDR_L, *hr = sd + SD_HDR_R;
    const int step = sd[SD_STEP];
    sd[SD_RECV_L] = P.has_left ? min(hl[0], P.halo_cap) : 0;
    sd[SD_RECV_R] = P.has_right ? min(hr[0], P.halo_cap) : 0;
    if (P.rebalance_every > 0 && step > 0 && step % P.rebalance_every == 0) {
        const int sx0 = sd[SD_SX0], sx1 = sd[SD_SX1], owned = sd[SD_OWNED];
        int n0 = sx0, n1 = sx1;
        if (P.has_left) n0 += shard_cut_move(hl[1], hl[3] - hl[2], owned, sx1 - sx0);
        if (P.has_right) n1 += shard_cut_move(owned, sx1 - sx0, hr[1], hr[3] - hr[2]);
        sd[SD_SX0] = n0; sd[SD_SX1] = n1;
    }
    sd[SD_STEP] = step + 1;
}

// After the sort: live count, owned range and the index ranges of the boundary layers to send, and the headers.
// send_layers = sgw + 1 (what the ghost band plus this step's migrants need) or, for the exchange that feeds a
// re-balancing step, sgw + 2 (the cut may then move by a layer); the host picks the graph variant by step number.
__global__ void k_shard_info(DevParams P, DevArrays S, int send_layers, int send_cap) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int32_t *sd = S.sd;
    const int layer = P.gy * P.gz;
    const int sx0 = sd[SD_SX0], sx1 = sd[SD_SX1];
    auto start_of_layer = [&](int L) {
        L = min(max(L, 0), P.gx);
        int c = L * layer;
        return c > 0 ? S.cell_end[c - 1] : 0;
    };
    const int n_live = S.cell_end[P.C - 1], n_sorted = S.cell_end[P.C];
    const int o0 = start_of_layer(sx0), o1 = start_of_layer(sx1);
    int l0 = o0, l1 = start_of_layer(min(sx0 + send_layers, sx1));
    int r0 = start_of_layer(max(sx1 - send_layers, sx0)), r1 = o1;
    if (!P.has_left) l1 = l0;
    if (!P.has_right) r0 = r1;
    uint32_t flags = 0u;
    if (l1 - l0 > send_cap) { l1 = l0 + send_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (r1 - r0 > send_cap) { r0 = r1 - send_cap; flags |= SPH_STATUS_HALO_CAPACITY; }
    if (n_sorted > P.n - 2 * P.halo_cap) flags |= SPH_STATUS_SHARD_CAPACITY;  // the sort ran into the receive regions
    if (flags) atomicOr(S.status, flags);
    sd[SD_N_LIVE] = n_live; sd[SD_N_SORTED] = n_sorted;
    sd[SD_OWNED] = o1 - o0; sd[SD_OWN0] = o0; sd[SD_OWN1] = o1;
    sd[SD_SEND_L0] = l0; sd[SD_SEND_L1] = l1; sd[SD_SEND_R0] = r0; sd[SD_SEND_R1] = r1;
    // densities are needed for the owned particles and the FIRST ghost layer of each side (the second one only
    // serves as neighbours of the first): one contiguous index range
    const int d0 = start_of_layer(sx0 - 1), d1 = start_of_layer(sx1 + 1);
    sd[SD_DENS0] = d0; sd[SD_DENS1] = d1;
    // ... and FIRST for everything within one layer of the send ranges (the boundary forces need exactly those), so
    // that the exchange can start before the interior densities: [d0, db_l1) and [db_r0, d1)
    int db_l1 = P.has_left ? start_of_layer(min(sx0 + send_layers + 1, sx1 + 1)) : d0;
    int db_r0 = P.has_right ? start_of_layer(max(sx1 - send_layers - 1, sx0 - 1)) : d1;
    db_r0 = max(db_r0, db_l1);
    sd[SD_DB_L1] = db_l1; sd[SD_DB_R0] = db_r0;
    sd[SD_FLAGS] = (int32_t)(*S.status);
    unsigned long long sent = ((unsigned long long)(uint32_t)sd[SD_SENT_HI] << 32) | (uint32_t)sd[SD_SENT_LO];
    sent += (unsigned long long)(l1 - l0) + (unsigned long long)(r1 - r0);
    sd[SD_SENT_LO] = (int32_t)(uint32_t)sent; sd[SD_SENT_HI] = (int32_t)(uint32_t)(sent >> 32);
    for (int side = 0; side < 2; ++side) {
        int32_t *h = S.stage_hdr[side];
        h[0] = side == 0 ? l1 - l0 : r1 - r0;
        h[1] = o1 - o0; h[2] = sx0; h[3] = sx1; h[4] = sd[SD_STEP];
    }
}

// The boundary pass of the force kernel wrote the advanced state of the send ranges into the staging (side, slot) =
// (0, i - l0) / (1, i - r0); after the interior densities are done it goes back into the packed arrays.
// copy_all = 1 (first exchange, no physics yet): pack the unchanged records instead.
__global__ void k_shard_apply(DevParams P, DevArrays S, int copy_all) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int side = blockIdx.y;
    const int32_t *sd = S.sd;
    const int b = side == 0 ? sd[SD_SEND_L0] : sd[SD_SEND_R0];
    const int e = side == 0 ? sd[SD_SEND_L1] : sd[SD_SEND_R1];
    if (s >= e - b) return;
    const int i = b + s;
    SPH_EMU_CHECK(s < P.halo_cap && i >= 0 && i < P.n);
    if (copy_all) {
        S.stage[side][0][s] = S.posm[i];
        S.stage[side][1][s] = S.veld[i];
        S.stage[side][2][s] = S.x0id[i];
        S.stage[side][3][s] = S.misc[i];
    } else {
        S.posm[i] = S.stage[side][0][s];  // (a particle inside both send ranges holds the same values in both stagings)
        S.veld[i] = S.stage[side][1][s];
    }
}

// In-place inclusive prefix sum over the per-cell counts (the reference's
// PrefixSumExecutor.run / scan_single_buffer.py:108-146, there a 3-level recursive scan with
// ~7 launches).  Here: ONE launch, decoupled look-back.  Each CTA takes a tile in arrival
// order, scans it with warp shuffles + shared memory, publishes {status, value} as one 64-bit
// word and resolves its exclusive prefix by looking back over predecessor tiles a warp at a time.
#ifndef SCAN_THREADS_VALUE
#define SCAN_THREADS_VALUE 512
#endif
#ifndef SCAN_IPT_VALUE
#define SCAN_IPT_VALUE 16
#endif
constexpr int SCAN_THREADS = SCAN_THREADS_VALUE;
constexpr int SCAN_IPT = SCAN_IPT_VALUE;  // multiple of 4 (128-bit loads); 8192 cells per tile: 58 tiles for 469 K cells --
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_IPT;  // one wave, at most two look-back rounds (was 2048 / 229 tiles)
#define SCAN_ST_AGG 1ull
#define SCAN_ST_PREFIX 2ull

__global__ void __launch_bounds__(SCAN_THREADS) k_scan(int32_t *__restrict__ data, int C,
                                                        unsigned long long *tile_state, int32_t *tile_counter) {
    pdl_wait();
    __shared__ int s_tile;
    __shared__ int s_warp[SCAN_THREADS / 32];
    __shared__ int s_excl;
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1);
    __syncthreads();
    const int tile = s_tile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int base = tile * SCAN_TILE + threadIdx.x * SCAN_IPT;

    int v[SCAN_IPT];
    if (base + SCAN_IPT <= C) {
#pragma unroll
        for (int q = 0; q < SCAN_IPT / 4; ++q) {
            int4 a = *reinterpret_cast<const int4 *>(data + base + 4 * q);
            v[4 * q] = a.x; v[4 * q + 1] = a.y; v[4 * q + 2] = a.z; v[4 * q + 3] = a.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_IPT; ++k) v[k] = (base + k < C) ? data[base + k] : 0;
    }
#pragma unroll
    for (int k = 1; k < SCAN_IPT; ++k) v[k] += v[k - 1];
    const int tsum = v[SCAN_IPT - 1];
    int incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = (lane < SCAN_THREADS / 32) ? s_warp[lane] : 0;
        int wi = w;
#pragma unroll
        for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        if (lane < SCAN_THREADS / 32) s_warp[lane] = wi - w;  // exclusive warp offsets
        const int agg = __shfl_sync(0xffffffffu, wi, SCAN_THREADS / 32 - 1);
        // ---- decoupled look-back ----
        volatile unsigned long long *st = tile_state;
        int excl = 0;
        if (tile > 0) {
            if (lane == 0) st[tile] = (SCAN_ST_AGG << 32) | (unsigned int)agg;
            int look = tile - 1;
            while (true) {
                int idx = look - lane;
                unsigned long long word = (SCAN_ST_PREFIX << 32);  // virtual tile -1: prefix 0
                if (idx >= 0) {
                    do { word = st[idx]; } while ((word >> 32) == 0ull);
                }
                unsigned int is_prefix = __ballot_sync(0xffffffffu, (word >> 32) == SCAN_ST_PREFIX);
                int val = (int)(unsigned int)(word & 0xffffffffull);
                int upto = is_prefix ? (__ffs(is_prefix) - 1) : 31;  // nearest tile holding a full prefix
                int contrib = (lane <= upto) ? val : 0;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
                excl += contrib;
                if (is_prefix) break;
                look -= 32;
            }
        }
        if (lane == 0) {
            st[tile] = (SCAN_ST_PREFIX << 32) | (unsigned int)(excl + agg);
            s_excl = excl;
        }
    }
    __syncthreads();
    const int off = s_excl + s_warp[warp] + (incl - tsum);
    if (base + SCAN_IPT <= C) {
#pragma unroll
        for (int q = 0; q < SCAN_IPT / 4; ++q)
            *reinterpret_cast<int4 *>(data + base + 4 * q) =
                make_int4(v[4 * q] + off, v[4 * q + 1] + off, v[4 * q + 2] + off, v[4 * q + 3] + off);
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_IPT; ++k)
            if (base + k < C) data[base + k] = v[k] + off;
    }
}

__global__ void k_bucket(DevParams P, DevArrays S) {
    pdl_wait();
    const int total = P.slab_on ? shard_input_total(S.sd) : P.n;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
        const int i = P.slab_on ? shard_input_index(P, S.sd, u) : u;
        int c = S.cid[i];
        int start = c > 0 ? S.cell_end[c - 1] : 0;
        S.perm[start + S.ticket[i]] = i;
    }
}

// The atomic tickets above give an arbitrary order inside a cell (as in the reference on a
// GPU, SURVEY Q7).  Ranking every bucket entry by its pre-sort index makes the result the
// STABLE counting sort -- the serial semantics of particle_system.py:325-330 -- so the sorted
// arrays are bit-reproducible and identical to the oracle's.
template <bool MOVE_ACC>
__global__ void k_rank_move(DevParams P, DevArrays S) {
    pdl_wait();
    const int total = P.slab_on ? S.cell_end[P.C] : P.n;  // sharded: P.n is the capacity, cell_end[C] the record count
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    int src = S.perm[t];
    int c = S.cid[src];
    int a = c > 0 ? S.cell_end[c - 1] : 0;
    int b = S.cell_end[c];
    int dst = t;  // trash bucket (slab mode): order is irrelevant and the bucket can be huge
    if (c < P.C) {
        int rank = 0;
        for (int u = a; u < b; ++u) rank += (S.perm[u] < src) ? 1 : 0;
        dst = a + rank;
    }
    float4 misc = S.misc[src];
    S.posm_n[dst] = S.posm[src];
    S.veld_n[dst] = S.veld[src];
    S.x0id_n[dst] = S.x0id[src];
    S.misc_n[dst] = misc;
    if (MOVE_ACC) S.acc_n[dst] = S.acc[src];  // the fused step overwrites every acceleration anyway
    S.grid_ids[dst] = c;
    int sid = __float_as_int(misc.w);
    if (sid >= 0) S.solid_slot[sid] = dst;
    }
}

// =====================================================================================
// simple pair kernels (v1): one thread per particle, 27-cell walk through L1.  They back the
// reference-named un-fused entry points and are the fallback for over-full neighbour lists.
// =====================================================================================

// Akinci boundary volumes (sph_base.py:91-113).  One WARP per solid particle: the lanes stride
// over the candidates of the 9 column runs and the partial sums are tree-reduced (a thread per
// particle left most of the GPU idle: a body has only a few thousand particles).
// SHARD (sharded steps with dynamic solids, after k_shard_solid_slots): only the solids in the owned layers and the
// first two ghost layers of each side -- the third one only serves as their neighbours.
template <bool SHARD = false>
__global__ void __launch_bounds__(128) k_boundary_volume(DevParams P, DevArrays S, int moving) {
    const int lane = threadIdx.x & 31;
    const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (s >= P.n_solid) return;  // warp-uniform
    const int i = S.solid_slot[s];
    if (SHARD && i < 0) return;  // not on this rank
    const uint32_t fl = __float_as_uint(S.misc[i].z);
    const bool dyn = (fl & FLAG_DYNAMIC) != 0;
    if (dyn != (moving != 0)) return;
    const float4 pi = S.posm[i];
    int ci, cj, ck;
    cell_of(P, pi.x, pi.y, pi.z, ci, cj, ck);
    if (SHARD && (ci < S.sd[SD_SX0] - 2 || ci >= S.sd[SD_SX1] + 2)) return;
    ci = min(max(ci, 0), P.gx - 1); cj = min(max(cj, 0), P.gy - 1); ck = min(max(ck, 0), P.gz - 1);
    const int k_lo = max(ck - 1, 0), k_hi = min(ck + 1, P.gz - 1);
    float part = 0.0f;
    for (int dx = -1; dx <= 1; ++dx) {
        int ni = ci + dx;
        if (ni < 0 || ni >= P.gx) continue;
        for (int dy = -1; dy <= 1; ++dy) {
            int nj = cj + dy;
            if (nj < 0 || nj >= P.gy) continue;
            int row = (ni * P.gy + nj) * P.gz;
            int j0 = __ldg(S.cell_end + max(row + k_lo - 1, 0));
            int j1 = __ldg(S.cell_end + row + k_hi);
            for (int j = j0 + lane; j < j1; j += 32) {
                float4 pj = __ldg(S.posm + j);
                float rx = pi.x - pj.x, ry = pi.y - pj.y, rz = pi.z - pj.z;
                float r2 = exact_r2(rx, ry, rz);
                if (r2 < P.h2 && j != i) {
                    uint32_t fj = __float_as_uint(__ldg(&S.misc[j].z));
                    if (!(fj & FLAG_FLUID)) part += w_cubic(P, sqrtf(r2));
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    // only .w changes; concurrent readers use .xyz only
    if (lane == 0) reinterpret_cast<float *>(S.posm + i)[3] = 1.0f / (P.w0 + part) * 3.0f;
}

// Densities (WCSPH.py:33-43).  FUSE_EOS additionally applies the clamp + Tait EOS of
// WCSPH.py:73-76 and initialises the accelerations of non-fluid particles (WCSPH.py:130-137),
// so the fused force pass can follow immediately.
template <bool FUSE_EOS>
__global__ void __launch_bounds__(128) k_density_simple(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float4 pi = S.posm[i];
    float4 mi = S.misc[i];
    uint32_t fl = __float_as_uint(mi.z);
    if (!(fl & FLAG_FLUID)) {
        bool dyn = (fl & FLAG_DYNAMIC) != 0;
        S.aux[i] = make_float4(S.veld[i].w, 0.0f, dyn ? -2.0f : -1.0f, 0.0f);
        if (FUSE_EOS) S.acc[i] = dyn ? make_float4(P.gx_, P.gy_, P.gz_, 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    float den = 0.0f;
    for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z,
                      [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
                          den += pj.w * w_cubic(P, sqrtf(r2));
                      });
    float rho = pi.w * P.w0;
    rho += den;
    rho *= P.rho0;
    float vol = mi.x / rho;  // m_j / rho_j with the UNCLAMPED density (viscosity, SURVEY Q4)
    if (FUSE_EOS) {
        float rc = fmaxf(rho, P.rho0);
        float p = tait_pressure(P, rc);
        reinterpret_cast<float *>(S.veld + i)[3] = rc;
        reinterpret_cast<float *>(S.misc + i)[1] = p;
        S.aux[i] = make_float4(vol, p / (rc * rc), mi.x, 0.0f);
    } else {
        reinterpret_cast<float *>(S.veld + i)[3] = rho;
        S.aux[i] = make_float4(vol, 0.0f, mi.x, 0.0f);
    }
}

// EOS loop of compute_pressure_forces (WCSPH.py:72-76), un-fused variant
__global__ void k_eos(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_FLUID)) return;
    float rc = fmaxf(S.veld[i].w, P.rho0);
    float p = tait_pressure(P, rc);
    reinterpret_cast<float *>(S.veld + i)[3] = rc;
    reinterpret_cast<float *>(S.misc + i)[1] = p;
    reinterpret_cast<float *>(S.aux + i)[1] = p / (rc * rc);
}

// Forces.  NP: compute_non_pressure_forces (WCSPH.py:88-140); PR: the gather loop of
// compute_pressure_forces (WCSPH.py:46-68,77-85).  NP && PR is the fused production pass.
template <bool NP, bool PR>
__global__ void __launch_bounds__(128) k_force_simple(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    float4 mi = S.misc[i];
    uint32_t fl = __float_as_uint(mi.z);
    if (!(fl & FLAG_FLUID)) {
        bool dyn = (fl & FLAG_DYNAMIC) != 0;
        if (NP && !PR) S.acc[i] = dyn ? make_float4(P.gx_, P.gy_, P.gz_, 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (PR && !NP && !dyn) S.acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;  // fused: initialised by the density pass
    }
    float4 pi = S.posm[i];
    float4 vi = S.veld[i];
    float4 ai = S.aux[i];
    const float dpi = ai.y;                      // p_i / rho_i^2
    const float dpi_solid = dpi + mi.y * P.inv_rho0sq;  // + p_i / rho0^2 (Akinci mirror, WCSPH.py:59)
    const float coh_i = P.sigma / mi.x;
    float npx = P.gx_, npy = P.gy_, npz = P.gz_;
    float prx = 0.f, pry = 0.f, prz = 0.f;
    for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z,
                      [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
                          float4 aj = __ldg(S.aux + j);
                          float r = sqrtf(r2);
                          float gs = gradw_scale(P, r);
                          if (aj.z > 0.0f) {  // fluid neighbour
                              if (NP) {
                                  float w = (r2 > P.d2) ? w_cubic(P, r) : P.w_diam;
                                  float c = coh_i * aj.z;
                                  npx -= c * rx * w; npy -= c * ry * w; npz -= c * rz * w;
                                  float4 vj = __ldg(S.veld + j);
                                  float vxy = (vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz;
                                  float sv = P.d_visc * aj.x * vxy / (r * r + P.visc_eps) * gs;
                                  npx += sv * rx; npy += sv * ry; npz += sv * rz;
                              }
                              if (PR) {
                                  float c = -P.rho0 * pj.w * (dpi + aj.y) * gs;
                                  prx += c * rx; pry += c * ry; prz += c * rz;
                              }
                          } else if (PR) {  // solid neighbour (Akinci 2012)
                              float c = -P.rho0 * pj.w * dpi_solid * gs;
                              float fx = c * rx, fy = c * ry, fz = c * rz;
                              prx += fx; pry += fy; prz += fz;
                              if (aj.z < -1.5f) {  // dynamic rigid: reaction, WCSPH.py:66-68
                                  float *a = reinterpret_cast<float *>(S.acc + j);
                                  atomicAdd(a + 0, -fx * P.rho0 / aj.x);
                                  atomicAdd(a + 1, -fy * P.rho0 / aj.x);
                                  atomicAdd(a + 2, -fz * P.rho0 / aj.x);
                              }
                          }
                      });
    if (NP && PR) {
        S.acc[i] = make_float4(npx + prx, npy + pry, npz + prz, 0.f);
    } else if (NP) {
        S.acc[i] = make_float4(npx, npy, npz, 0.f);
    } else {
        float4 a = S.acc[i];
        S.acc[i] = make_float4(a.x + prx, a.y + pry, a.z + prz, 0.f);
    }
}

// =====================================================================================
// integration and domain walls
// =====================================================================================
__device__ __forceinline__ void wall_clamp(const DevParams &P, float4 &p, float4 &v) {
    // sph_base.py:118-123,149-179
    float nx = 0.f, ny = 0.f, nz = 0.f;
    float px = p.x, py = p.y, pz = p.z;
    if (px > P.hi_x) { nx += 1.0f; p.x = P.hi_x; }
    if (px <= P.pad) { nx += -1.0f; p.x = P.pad; }
    if (py > P.hi_y) { ny += 1.0f; p.y = P.hi_y; }
    if (py <= P.pad) { ny += -1.0f; p.y = P.pad; }
    if (pz > P.hi_z) { nz += 1.0f; p.z = P.hi_z; }
    if (pz <= P.pad) { nz += -1.0f; p.z = P.pad; }
    float len = sqrtf(nx * nx + ny * ny + nz * nz);
    if (len > 1e-6f) {
        nx /= len; ny /= len; nz /= len;
        float f = (1.0f + 0.5f) * (v.x * nx + v.y * ny + v.z * nz);
        v.x -= f * nx; v.y -= f * ny; v.z -= f * nz;
    }
}

// advect (WCSPH.py:143-149); CLAMP_FLUID fuses enforce_boundary_3D(material_fluid), which only
// touches fluid particles and therefore commutes with the rigid-body solve in between.
template <bool CLAMP_FLUID>
__global__ void k_advect(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC) || (fl & FLAG_GHOST)) return;
    if (P.slab_on && i >= S.sd[SD_N_LIVE]) return;
    float4 p = S.posm[i], v = S.veld[i], a = S.acc[i];
    v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    if (CLAMP_FLUID && (fl & FLAG_FLUID)) wall_clamp(P, p, v);
    S.posm[i] = p;
    S.veld[i] = v;
}

__global__ void k_enforce_boundary(DevParams P, DevArrays S, int particle_type) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    if (P.slab_on && (i < S.sd[SD_OWN0] || i >= S.sd[SD_OWN1])) return;  // sharded DFSPH: owned particles only
    uint32_t fl = __float_as_uint(S.misc[i].z);
    int mat = (fl & FLAG_FLUID) ? SPH_MATERIAL_FLUID : SPH_MATERIAL_SOLID;
    if (mat != particle_type || !(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i];
    wall_clamp(P, p, v);
    S.posm[i] = p;
    S.veld[i] = v;
}

struct RigidBodyDev {
    int32_t object_id, solid_begin, solid_end;
    float rest_cm[3];
    float R[9];   // rotation of the last solve_constraints
    float cm[3];  // centre of mass of the last solve_constraints
};

// enforce_boundary_3D(material_solid) restricted to the solid list (cheaper than a full sweep).  reps > 1 with
// skip_bodies: the fused step applies the n clamps of the reference's body loop to the dynamic solids that belong to NO
// shape-matched body here (k_rigid does it for the bodies' own particles).
// SHARD: owned solids only (the slot map of k_shard_solid_slots).
template <bool SHARD = false>
__global__ void k_enforce_boundary_solid(DevParams P, DevArrays S, int reps, const RigidBodyDev *skip_bodies, int n_skip) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.n_solid) return;
    for (int b = 0; b < n_skip; ++b)
        if (s >= skip_bodies[b].solid_begin && s < skip_bodies[b].solid_end) return;
    int i = S.solid_slot[s];
    if (SHARD && (i < S.sd[SD_OWN0] || i >= S.sd[SD_OWN1])) return;  // -1 (not on this rank) or a ghost
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i];
    for (int r = 0; r < reps; ++r) wall_clamp(P, p, v);
    S.posm[i] = p;
    S.veld[i] = v;
}

// =====================================================================================
// rigid bodies: shape matching (sph_base.py:182-222).  One CTA per call, fixed-order tree
// reductions (deterministic), polar decomposition in fp64 on one thread.
// =====================================================================================
constexpr int RIGID_THREADS = 1024;

template <int NV>
__device__ __forceinline__ void block_reduce(float (&v)[NV], float *smem /* [32 * NV] */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    __syncthreads();
    if (lane == 0)
        for (int k = 0; k < NV; ++k) smem[warp * NV + k] = v[k];
    __syncthreads();
    const int nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        float t = (lane < nw) ? smem[lane * NV + k] : 0.0f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        v[k] = t;  // every thread holds the total
    }
}

// Rotation factor of the polar decomposition A = R S (what ti.polar_decompose returns for R):
// scaled Newton iteration X <- (g X + X^-T / g) / 2 in fp64 on one thread; 3 divisions and 2 square
// roots per iteration (fp64 latency is what this single thread pays for), ~8 iterations.
__device__ void polar_rotation_f64(const double A[9], double R[9], bool &ok) {
    double X[9];
    for (int i = 0; i < 9; ++i) X[i] = A[i];
    ok = true;
    for (int it = 0; it < 100; ++it) {
        double c[9];  // cofactors: X^-T = c / det
        c[0] = X[4] * X[8] - X[5] * X[7]; c[1] = X[5] * X[6] - X[3] * X[8]; c[2] = X[3] * X[7] - X[4] * X[6];
        c[3] = X[2] * X[7] - X[1] * X[8]; c[4] = X[0] * X[8] - X[2] * X[6]; c[5] = X[1] * X[6] - X[0] * X[7];
        c[6] = X[1] * X[5] - X[2] * X[4]; c[7] = X[2] * X[3] - X[0] * X[5]; c[8] = X[0] * X[4] - X[1] * X[3];
        double det = X[0] * c[0] + X[1] * c[1] + X[2] * c[2];
        if (fabs(det) < 1e-300) { ok = false; break; }
        const double inv_det = 1.0 / det;
        double nx = 0, ni = 0;
        for (int i = 0; i < 9; ++i) { c[i] *= inv_det; nx += X[i] * X[i]; ni += c[i] * c[i]; }
        const double gamma = sqrt(sqrt(ni / nx));  // Frobenius-norm scaling
        const double inv_gamma = 1.0 / gamma;
        double diff = 0;
        for (int i = 0; i < 9; ++i) {
            double y = 0.5 * (gamma * X[i] + c[i] * inv_gamma);
            diff += (y - X[i]) * (y - X[i]);
            X[i] = y;
        }
        if (diff < 1e-30) break;
    }
    for (int i = 0; i < 9; ++i) R[i] = X[i];
    // The iteration converges to the ORTHOGONAL polar factor Q, det Q = sign(det A).  ti.polar_decompose takes R
    // from an SVD whose U and V are proper rotations (the smallest singular value carries the sign), i.e.
    // R = Q (I - 2 v v^T) with v the eigenvector of S = Q^T A of smallest eigenvalue when det A < 0 (a collapsed
    // or inverted body).  Cyclic Jacobi on the symmetric 3x3 S; only that rare case pays for it.
    const double detA = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    if (ok && detA < 0.0) {
        double S[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) S[3 * r + c] = X[r] * A[c] + X[3 + r] * A[3 + c] + X[6 + r] * A[6 + c];  // Q^T A
        for (int r = 0; r < 3; ++r)
            for (int c = r + 1; c < 3; ++c) S[3 * r + c] = S[3 * c + r] = 0.5 * (S[3 * r + c] + S[3 * c + r]);
        for (int sweep = 0; sweep < 12; ++sweep) {
            for (int p = 0; p < 2; ++p)
                for (int q = p + 1; q < 3; ++q) {
                    const double apq = S[3 * p + q];
                    if (fabs(apq) < 1e-300) continue;
                    const double th = 0.5 * (S[3 * q + q] - S[3 * p + p]) / apq;
                    const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                    const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
                    for (int k = 0; k < 3; ++k) {  // S <- S J
                        const double skp = S[3 * k + p], skq = S[3 * k + q];
                        S[3 * k + p] = cs * skp - sn * skq; S[3 * k + q] = sn * skp + cs * skq;
                    }
                    for (int k = 0; k < 3; ++k) {  // S <- J^T S,  V <- V J
                        const double spk = S[3 * p + k], sqk = S[3 * q + k];
                        S[3 * p + k] = cs * spk - sn * sqk; S[3 * q + k] = sn * spk + cs * sqk;
                        const double vkp = V[3 * k + p], vkq = V[3 * k + q];
                        V[3 * k + p] = cs * vkp - sn * vkq; V[3 * k + q] = sn * vkp + cs * vkq;
                    }
                }
        }
        int m = 0;
        if (S[4] < S[3 * m + m]) m = 1;
        if (S[8] < S[3 * m + m]) m = 2;
        const double v[3] = {V[m], V[3 + m], V[6 + m]};
        for (int r = 0; r < 3; ++r) {
            const double qv = X[3 * r] * v[0] + X[3 * r + 1] * v[1] + X[3 * r + 2] * v[2];
            for (int c = 0; c < 3; ++c) R[3 * r + c] = X[3 * r + c] - 2.0 * qv * v[c];
        }
    }
}

// mode 0: compute_com -> out[3];  mode 1: store rest cm;  mode 2: solve_constraints.
// One gather pass accumulates the raw moments  M = sum m,  X = sum m x,  Q = sum m q,  XQ = sum m x (x) q
// (q = x_0 - rest_cm); then  cm = X / M  and  A = sum m (x - cm) (x) q = XQ - cm (x) Q  (sph_base.py:182-211).
// n_step_bodies > 0 (fused step, mode 2, one CTA per body = blockIdx.x): the reference solves the bodies one after
// the other and clamps ALL dynamic solid particles to the walls after each solve (sph_base.py:247-260), i.e. a
// particle of body b is clamped b times before its body is solved and n - b times after.  The bodies' particle
// sets are disjoint and a clamp only looks at the particle itself, so the same sequence runs here per body in ONE
// launch (3 bodies: 6 launches -> 2, bit-identical).
__global__ void __launch_bounds__(RIGID_THREADS) k_rigid(DevParams P, DevArrays S, RigidBodyDev *bodies, int body,
                                                          int mode, float *out, int n_step_bodies) {
    __shared__ float red[32 * 16];
    __shared__ float s_R[9];
    if (n_step_bodies > 0) body = blockIdx.x;
    const int pre_clamps = n_step_bodies > 0 ? body : 0, post_clamps = n_step_bodies > 0 ? n_step_bodies - body : 0;
    RigidBodyDev *B = bodies + body;
    const int b0 = B->solid_begin, b1 = B->solid_end;
    const float r0 = B->rest_cm[0], r1 = B->rest_cm[1], r2 = B->rest_cm[2];
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int s = b0 + threadIdx.x; s < b1; s += blockDim.x) {
        int i = S.solid_slot[s];
        uint32_t fl = __float_as_uint(S.misc[i].z);
        if (!(fl & FLAG_DYNAMIC)) continue;  // compute_com counts dynamic rigid particles only (Q8)
        float4 p = S.posm[i], x0 = S.x0id[i];
        if (pre_clamps > 0) {  // the clamps the earlier bodies' iterations applied to this particle
            float4 v = S.veld[i];
            for (int r = 0; r < pre_clamps; ++r) wall_clamp(P, p, v);
            S.posm[i] = p;
            S.veld[i] = v;
        }
        float mass = P.m_V0 * S.veld[i].w;
        float q[3] = {x0.x - r0, x0.y - r1, x0.z - r2};
        float x[3] = {p.x, p.y, p.z};
        acc[0] += mass;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            acc[1 + r] += mass * x[r];
            acc[4 + r] += mass * q[r];
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[7 + 3 * r + c] += mass * x[r] * q[c];
        }
    }
    block_reduce<16>(acc, red);
    const float cmx = acc[1] / acc[0], cmy = acc[2] / acc[0], cmz = acc[3] / acc[0];
    if (mode == 0) {
        if (threadIdx.x == 0) { out[0] = cmx; out[1] = cmy; out[2] = cmz; }
        return;
    }
    if (mode == 1) {
        if (threadIdx.x == 0) { B->rest_cm[0] = cmx; B->rest_cm[1] = cmy; B->rest_cm[2] = cmz; }
        return;
    }
    if (threadIdx.x == 0) {
        const float cm[3] = {cmx, cmy, cmz};
        double Ad[9], Rd[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Ad[3 * r + c] = (double)acc[7 + 3 * r + c] - (double)cm[r] * (double)acc[4 + c];
        bool ok;
        polar_rotation_f64(Ad, Rd, ok);
        if (!ok) atomicOr(S.status, SPH_STATUS_BAD_POLAR);
        bool all_small = true;
        float Rf[9];
        for (int k = 0; k < 9; ++k) { Rf[k] = (float)Rd[k]; if (!(fabsf(Rf[k]) < 1e-6f)) all_small = false; }
        if (all_small) { for (int k = 0; k < 9; ++k) Rf[k] = (k % 4 == 0) ? 1.0f : 0.0f; }
        for (int k = 0; k < 9; ++k) { s_R[k] = Rf[k]; B->R[k] = Rf[k]; if (out) out[k] = Rf[k]; }
        B->cm[0] = cmx; B->cm[1] = cmy; B->cm[2] = cmz;
    }
    __syncthreads();
    for (int s = b0 + threadIdx.x; s < b1; s += blockDim.x) {
        int i = S.solid_slot[s];
        uint32_t fl = __float_as_uint(S.misc[i].z);
        if (!(fl & FLAG_DYNAMIC)) continue;
        float4 p = S.posm[i], x0 = S.x0id[i];
        float q0 = x0.x - r0, q1 = x0.y - r1, q2 = x0.z - r2;
        float gx = cmx + (s_R[0] * q0 + s_R[1] * q1 + s_R[2] * q2);
        float gy = cmy + (s_R[3] * q0 + s_R[4] * q1 + s_R[5] * q2);
        float gz = cmz + (s_R[6] * q0 + s_R[7] * q1 + s_R[8] * q2);
        p.x += (gx - p.x) * 1.0f; p.y += (gy - p.y) * 1.0f; p.z += (gz - p.z) * 1.0f;
        if (post_clamps > 0) {  // this body's own clamp and those of the later bodies' iterations
            float4 v = S.veld[i];
            for (int r = 0; r < post_clamps; ++r) wall_clamp(P, p, v);
            S.veld[i] = v;
        }
        S.posm[i] = p;
    }
}

// =====================================================================================
// Production pair kernels.  History: DESIGN.md section 3.1.
//
//  * The density pass scans the 27-cell candidates once per step and appends the accepted pairs
//    to a per-particle neighbour list (reference visiting order); the force pass is a dense loop
//    over that list (v1 executed the 80-instruction hit path under a ~15 % per-lane hit rate).
//  * Candidate windows are staged by TMA: each WARP copies, per (dx, dy) column, the union of its
//    lanes' candidate ranges -- one contiguous run of the sorted posm array -- into shared memory
//    with one cp.async.bulk (SASS UBLKCP) completing on an mbarrier, double-buffered over the 9
//    columns; lanes scan their own sub-range with LDS.128.
//  * The scan is branch-free: 32 candidates at a time into a per-lane hit bitmask, then the set
//    bits are flushed (list append + density contribution straight from the staged window).
//  * The force pass gathers 2 x 16 B per neighbour (uniform fluids) in batches of 4 with all
//    loads of a batch issued before any arithmetic, and integrates the particle in its epilogue.
//  Particles with more than NBR_CAP neighbours fall back to the v1 full scan in the same kernels.
// =====================================================================================
struct ForceAcc {
    float npx, npy, npz, prx, pry, prz;
};

// one accepted pair of the fused force pass (WCSPH.py:46-68 and 88-125); aj / vj already loaded
__device__ __forceinline__ void force_pair_pre(const DevParams &P, const DevArrays &S, ForceAcc &A, int j, float rx,
                                               float ry, float rz, float r2, float mVj, const float4 &aj,
                                               const float4 &vj, const float4 &vi, float dpi, float dpi_solid,
                                               float coh_i) {
    float r, inv_r;
    fast_norm(r2, r, inv_r);
    float gs = gradw_scale_fast(P, r, inv_r);
    if (aj.z > 0.0f) {  // fluid neighbour
        float w = (r2 > P.d2) ? w_cubic(P, r) : P.w_diam;
        float c = coh_i * aj.z;
        A.npx -= c * rx * w; A.npy -= c * ry * w; A.npz -= c * rz * w;
        float vxy = (vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz;
        float sv = __fdividef(P.d_visc * aj.x * vxy, r * r + P.visc_eps) * gs;
        A.npx += sv * rx; A.npy += sv * ry; A.npz += sv * rz;
        float cp = -P.rho0 * mVj * (dpi + aj.y) * gs;
        A.prx += cp * rx; A.pry += cp * ry; A.prz += cp * rz;
    } else {  // solid neighbour (Akinci 2012)
        float cp = -P.rho0 * mVj * dpi_solid * gs;
        float fx = cp * rx, fy = cp * ry, fz = cp * rz;
        A.prx += fx; A.pry += fy; A.prz += fz;
        if (aj.z < -1.5f) {  // dynamic rigid: reaction, WCSPH.py:66-68
            float *a = reinterpret_cast<float *>(S.acc + j);
            atomicAdd(a + 0, -fx * P.rho0 / aj.x);
            atomicAdd(a + 1, -fy * P.rho0 / aj.x);
            atomicAdd(a + 2, -fz * P.rho0 / aj.x);
        }
    }
}

// ---- staging windows (the TMA / mbarrier primitives live in sph_ptx.cuh) ----
#ifndef WIN_CAP_VALUE
#define WIN_CAP_VALUE 128
#endif
constexpr int WIN_CAP = WIN_CAP_VALUE;   // particles per staged window (2 KB); longer windows scan global memory
#ifndef DENS_WARPS_VALUE
#define DENS_WARPS_VALUE 4
#endif
constexpr int DENS_WARPS = DENS_WARPS_VALUE;

// Branch-free distance test of up to 32 candidates starting at jb.  d = |r|^2 - h^2 comes straight
// out of a 3-FFMA chain and its sign bit is funnel-shifted into the mask (one SHF per candidate),
// so the FIRST candidate ends up in the HIGHEST of the `len` valid bits: candidate u <-> bit len-1-u.
template <bool FROM_SMEM>
__device__ __forceinline__ uint32_t scan_chunk(const DevParams &P, const float4 *__restrict__ src, int jb, int len,
                                               int j_last, float xi, float yi, float zi) {
    uint32_t m = 0u;
    int done = 0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        if (g * 8 < len) {
#pragma unroll
            for (int u = g * 8; u < g * 8 + 8; ++u) {
                float4 pj = FROM_SMEM ? src[jb + u] : __ldg(src + min(jb + u, j_last));
                float rx = xi - pj.x, ry = yi - pj.y, rz = zi - pj.z;
                float d = fmaf(rz, rz, fmaf(ry, ry, fmaf(rx, rx, -P.h2_scan)));  // conservative prefilter
                m = __funnelshift_l(__float_as_uint(d), m, 1);
            }
            done = g * 8 + 8;
        }
    }
    return m >> (done - len);  // drop the padding candidates of the last group
}

// Densities (WCSPH.py:33-43) + clamp and Tait EOS (WCSPH.py:73-76) + neighbour-list build +
// initial accelerations of non-fluid particles (WCSPH.py:130-137).
// INLINE_W: the density contribution of a hit is taken from the staged window while flushing the
// bitmask; otherwise a second dense loop re-gathers the neighbours from global memory.
#ifndef DENS_MIN_BLOCKS
#define DENS_MIN_BLOCKS 8  // H100 sweep of 7-10 blocks/SM: 8 is fastest on dragon_bath and armadillo (DESIGN.md 3.1)
#endif
// FASTW (with INLINE_W): the branch-free spline_w_norm() with the 2k factor applied once per particle;
// DFSPH keeps the reference's piecewise form (its solver loops count iterations against the oracle).
// split_mode (sharded steps): 1 = only the particles within one layer of the send ranges, 2 = only the others,
// 0 = all that need a density.
template <bool INLINE_W, bool FASTW>
__global__ void __launch_bounds__(DENS_WARPS * 32, DENS_MIN_BLOCKS) k_density_tma(DevParams P, DevArrays S, int split_mode) {
    pdl_wait();
    __shared__ __align__(128) float4 s_win[DENS_WARPS][2][WIN_CAP + 32];
    __shared__ __align__(8) uint64_t s_bar[DENS_WARPS][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { mbar_init(&s_bar[warp][0], 1); mbar_init(&s_bar[warp][1], 1); }
    mbar_fence_init();
    __syncwarp();
    uint32_t phase = 0u;  // bit b = parity of the next completion of barrier b (persists across the tiles of a block)

    // one tile = blockDim.x consecutive particles starting at i - threadIdx.x; i_end bounds the particles that need
    // a density
    auto tile = [&](const int i) {
    bool live = i < P.n;
    if (P.slab_on) {
        // sharded steps: the grid covers the capacity (the hardware block scheduler balanced better than a persistent
        // tile loop when both were tried); only owned particles
        // + the first ghost layer per side -- one index range of the device-resident step state -- need a density
        const int32_t *sd = S.sd;
        live = i >= sd[SD_DENS0] && i < sd[SD_DENS1];
        if (split_mode) {
            const bool boundary = i < sd[SD_DB_L1] || i >= sd[SD_DB_R0];
            live = live && ((split_mode == 1) == boundary);
        }
    }
    float4 pi = make_float4(0.f, 0.f, 0.f, 0.f), mi = pi;
    uint32_t fl = 0;
    if (live) { pi = S.posm[i]; mi = S.misc[i]; fl = __float_as_uint(mi.z); }
    const bool fluid = live && (fl & FLAG_FLUID);
    if (live && !fluid) {
        bool dyn = (fl & FLAG_DYNAMIC) != 0;
        float4 vb = S.veld[i];
        S.aux[i] = make_float4(vb.w, 0.0f, dyn ? -2.0f : -1.0f, 0.0f);
        if (!P.dfsph) S.acc[i] = dyn ? make_float4(P.gx_, P.gy_, P.gz_, 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
        S.nbr_cnt[i] = 0;
        if (P.uniform_fluid) {
            S.fpv[2 * (size_t)i] = pi;  // w = m_V of the boundary particle
            S.fpv[2 * (size_t)i + 1] = make_float4(vb.x, vb.y, vb.z, dyn ? -vb.w : -__int_as_float(0x7f800000));
        }
    }
    if (__ballot_sync(0xffffffffu, fluid) == 0u) return;  // warp-uniform

    int ci = 0, cj = 0, ck = 0;
    cell_of(P, pi.x, pi.y, pi.z, ci, cj, ck);
    ci = min(max(ci, 0), P.gx - 1); cj = min(max(cj, 0), P.gy - 1); ck = min(max(ck, 0), P.gz - 1);
    const int k_lo = max(ck - 1, 0), k_hi = min(ck + 1, P.gz - 1);
    // per-lane candidate range of the p-th visited column c = (dx + 1) * 3 + (dy + 1) (DevParams::col_order)
    auto col_range = [&](int p, int &j0, int &j1) {
        const int c = (int)((P.col_order >> (4 * p)) & 15ull);
        int ni = ci + c / 3 - 1, nj = cj + c % 3 - 1;
        j0 = 0; j1 = 0;
        if (fluid && ni >= 0 && ni < P.gx && nj >= 0 && nj < P.gy) {
            int row = (ni * P.gy + nj) * P.gz;
            j0 = __ldg(S.cell_end + max(row + k_lo - 1, 0));
            j1 = __ldg(S.cell_end + row + k_hi);
        }
    };
    // warp-uniform window [J0, J1) and its staging into buffer b.  Returns 0 = empty, 1 = staged
    // (wait on the barrier), 2 = longer than WIN_CAP: scan global memory directly.
    auto stage = [&](int j0, int j1, int b, int &J0, int &J1) -> int {
        bool ne = j1 > j0;
        J0 = __reduce_min_sync(0xffffffffu, ne ? j0 : 0x7fffffff);
        J1 = __reduce_max_sync(0xffffffffu, ne ? j1 : 0);
        if (J1 <= J0) return 0;
        if (J1 - J0 > WIN_CAP) return 2;
        if (lane == 0) {
            uint32_t bytes = (uint32_t)(J1 - J0) * 16u;
            mbar_expect_tx(&s_bar[warp][b], bytes);
            tma_bulk_g2s(&s_win[warp][b][0], S.posm + J0, bytes, &s_bar[warp][b]);
        }
        return 1;
    };

    int cnt = 0;
    float den = 0.0f;
    uint32_t widx = (uint32_t)(fluid ? i : 0);  // index of the next list slot
    const uint32_t widx_cap = widx + (uint32_t)(NBR_CAP - 1) * (uint32_t)S.npad;  // last row
    auto flush = [&](uint32_t m, int jb, int len, const float4 *src, bool smem) {
        if ((uint32_t)(i - jb) < (uint32_t)len) m &= ~(1u << (len - 1 - (i - jb)));  // p_i != p_j
        while (m) {
            int hb = 31 - __clz(m);  // highest set bit = earliest candidate: keeps the reference order
            m &= ~(1u << hb);
            int b = len - 1 - hb;
            float4 pj = smem ? src[jb + b] : __ldg(src + jb + b);
            float rx = pi.x - pj.x, ry = pi.y - pj.y, rz = pi.z - pj.z;
            float r2 = exact_r2(rx, ry, rz);
            if (r2 < P.h2) {  // the exact `norm() < h` of the reference; the scan only pre-filters
                SPH_EMU_CHECK((uint64_t)widx < (uint64_t)NBR_CAP * (uint64_t)S.npad && jb + b >= 0 && jb + b < P.n);
                S.nbr_list[widx] = jb + b;  // beyond NBR_CAP the last row is overwritten (flagged below)
                widx = min(widx + (uint32_t)S.npad, widx_cap);
                ++cnt;
                if (INLINE_W && FASTW) {
                    den = fmaf(pj.w, spline_w_norm(P, r2), den);
                } else if (INLINE_W) {
                    float r, inv_r;
                    fast_norm(r2, r, inv_r);
                    den += pj.w * w_cubic(P, r);
                }
            }
        }
    };

    int j0n, j1n, J0n, J1n;
    col_range(0, j0n, j1n);
    int mode_n = stage(j0n, j1n, 0, J0n, J1n);
    for (int c = 0; c < 9; ++c) {
        const int b = c & 1;
        const int j0 = j0n, j1 = j1n, J0 = J0n, mode = mode_n;
        if (c + 1 < 9) {
            col_range(c + 1, j0n, j1n);
            __syncwarp();  // every lane is done reading buffer b^1 (column c - 1)
            mode_n = stage(j0n, j1n, b ^ 1, J0n, J1n);
        }
        if (mode == 1) {
            mbar_wait(&s_bar[warp][b], (phase >> b) & 1u);
            phase ^= 1u << b;
            const float4 *w = &s_win[warp][b][0] - J0;
            for (int jb = j0; jb < j1; jb += 32) {
                const int len = min(32, j1 - jb);
                SPH_EMU_CHECK(jb >= J0 && jb + len - J0 <= WIN_CAP);  // inside the staged window
                flush(scan_chunk<true>(P, w, jb, len, 0, pi.x, pi.y, pi.z), jb, len, w, true);
            }
        } else if (mode == 2) {
            for (int jb = j0; jb < j1; jb += 32) {
                const int len = min(32, j1 - jb);
                flush(scan_chunk<false>(P, S.posm, jb, len, j1 - 1, pi.x, pi.y, pi.z), jb, len, S.posm, false);
            }
        }
    }
    if (!fluid) return;

    if (cnt <= NBR_CAP) {
        S.nbr_cnt[i] = cnt;
        // pad the list to a multiple of LIST_PAD with the particle itself: the batched force pass then
        // loads whole batches without per-entry predicates (a self pair contributes exactly zero)
        for (int k = cnt; k % LIST_PAD; ++k) { S.nbr_list[widx] = i; widx += (uint32_t)S.npad; }
        if (!INLINE_W) {
            const size_t stride = (size_t)S.npad;
            const int32_t *lq = S.nbr_list + i;
            for (int k0 = 0; k0 < cnt; k0 += 4) {
                float4 pj[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    int j = (k0 + u < cnt) ? lq[(size_t)(k0 + u) * stride] : i;
                    pj[u] = __ldg(S.posm + j);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float rx = pi.x - pj[u].x, ry = pi.y - pj[u].y, rz = pi.z - pj[u].z;
                    float r2 = rx * rx + ry * ry + rz * rz;
                    float r, inv_r;
                    fast_norm(r2, r, inv_r);
                    float wv = pj[u].w * w_cubic(P, r);
                    den += (k0 + u < cnt) ? wv : 0.0f;
                }
            }
        }
    } else {
        S.nbr_cnt[i] = NBR_OVERFLOW;
        if (!INLINE_W) {
            for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z,
                              [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
                                  den += pj.w * w_cubic(P, sqrtf(r2));
                              });
        }
    }
    float rho = pi.w * P.w0;
    rho = (INLINE_W && FASTW) ? fmaf(den, P.k2_w, rho) : rho + den;
    rho *= P.rho0;
    float vol = mi.x / rho;  // m_j / rho_j with the UNCLAMPED density (viscosity, SURVEY Q4)
    if (P.dfsph) {  // DFSPH.py:39-47: plain density, no clamp, no EOS
        reinterpret_cast<float *>(S.veld + i)[3] = rho;
        S.aux[i] = make_float4(vol, 0.0f, mi.x, 0.0f);
        return;
    }
    float rc = fmaxf(rho, P.rho0);
    float p = tait_pressure(P, rc);
    float dp = p / (rc * rc);
    reinterpret_cast<float *>(S.veld + i)[3] = rc;
    reinterpret_cast<float *>(S.misc + i)[1] = p;
    S.aux[i] = make_float4(vol, dp, mi.x, 0.0f);
    if (P.uniform_fluid) {
        float4 vb = S.veld[i];
        S.fpv[2 * (size_t)i] = make_float4(pi.x, pi.y, pi.z, vol);
        S.fpv[2 * (size_t)i + 1] = make_float4(vb.x, vb.y, vb.z, dp);
    }
    };  // tile
    tile(blockIdx.x * blockDim.x + threadIdx.x);
}

// Fused force pass, general particle masses: 3 x 16 B gathered per neighbour.
template <int B, int THREADS>
__global__ void __launch_bounds__(THREADS) k_force_general(DevParams P, DevArrays S) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    if (P.slab_on && i >= S.sd[SD_N_LIVE]) return;
    float4 mi = S.misc[i];
    uint32_t fl = __float_as_uint(mi.z);
    if (!(fl & FLAG_FLUID)) return;  // initialised by k_density_tma
    if (fl & FLAG_GHOST) return;     // ghosts are neighbours only
    float4 pi = S.posm[i];
    float4 vi = S.veld[i];
    float4 ai = S.aux[i];
    const float dpi = ai.y;                              // p_i / rho_i^2
    const float dpi_solid = dpi + mi.y * P.inv_rho0sq;   // + p_i / rho0^2 (Akinci mirror, WCSPH.py:59)
    const float coh_i = P.sigma / mi.x;
    ForceAcc A = {P.gx_, P.gy_, P.gz_, 0.f, 0.f, 0.f};
    const int cnt = S.nbr_cnt[i];
    if (cnt != NBR_OVERFLOW) {
        const int32_t *lp = S.nbr_list + i;
        const size_t stride = (size_t)S.npad;
        for (int k0 = 0; k0 < cnt; k0 += B) {
            int j[B];  // the tail is padded with i itself: its pair terms are exactly zero
#pragma unroll
            for (int u = 0; u < B; ++u) j[u] = (k0 + u < cnt) ? lp[(size_t)(k0 + u) * stride] : i;
            float4 pj[B], aj[B], vj[B];
#pragma unroll
            for (int u = 0; u < B; ++u) {
                pj[u] = __ldg(S.posm + j[u]);
                aj[u] = __ldg(S.aux + j[u]);
                vj[u] = __ldg(S.veld + j[u]);
            }
#pragma unroll
            for (int u = 0; u < B; ++u) {
                float rx = pi.x - pj[u].x, ry = pi.y - pj[u].y, rz = pi.z - pj[u].z;
                float r2 = rx * rx + ry * ry + rz * rz;
                force_pair_pre(P, S, A, j[u], rx, ry, rz, r2, pj[u].w, aj[u], vj[u], vi, dpi, dpi_solid, coh_i);
            }
        }
    } else {
        for_all_neighbors(P, S.posm, S.cell_end, i, pi.x, pi.y, pi.z,
                          [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
                              force_pair_pre(P, S, A, j, rx, ry, rz, r2, pj.w, __ldg(S.aux + j), __ldg(S.veld + j), vi,
                                             dpi, dpi_solid, coh_i);
                          });
    }
    S.acc[i] = make_float4(A.npx + A.prx, A.npy + A.pry, A.npz + A.prz, 0.f);
}

// one accepted pair, uniform-fluid packing (see DevArrays::fpv).  Per-thread constants fold the spline
// normalisations: grad W = K1 * G * r_vec, W = k2 * wn (spline_pair), so that cohesion, viscosity and
// the pressure term (WCSPH.py:100-127, 55-85) collapse into ONE scalar s with a_i += s * r_vec.
struct PackedConst {
    float cohk;  // sigma / m_i * m_j * 2k  (cohesion uses W(max(r, d)), WCSPH.py:104-109)
    float cp;    // rho0 * m_V of a fluid neighbour
    float cps;   // rho0 * (p_i / rho_i^2 + p_i / rho0^2)  (solid neighbour, WCSPH.py:63)
};
// REACT = false (sharded steps): no reaction scatter onto dynamic solids; k_shard_reactions gathers the same terms.
template <bool REACT = true>
__device__ __forceinline__ void force_pair_packed(const DevParams &P, const DevArrays &S, ForceAcc &A, int j, float rx,
                                                  float ry, float rz, float r2, const float4 &pj, const float4 &vj,
                                                  const float4 &vi, float dpi, const PackedConst &K) {
    float wn, G;
    spline_pair(P, r2, wn, G);
    const float g1 = G * P.k1_grad;
    if (vj.w >= 0.0f) {  // fluid neighbour: pj.w = m_j / rho_j, vj.w = p_j / rho_j^2
        wn = (r2 > P.d2) ? wn : P.wd_norm;
        float vxy = (vi.x - vj.x) * rx + (vi.y - vj.y) * ry + (vi.z - vj.z) * rz;
        float q1 = pj.w * vxy * rcp_ftz(r2 + P.visc_eps);
        float tt = fmaf(q1, P.d_visc, -K.cp * (dpi + vj.w));
        float s = fmaf(g1, tt, -K.cohk * wn);
        A.npx = fmaf(s, rx, A.npx); A.npy = fmaf(s, ry, A.npy); A.npz = fmaf(s, rz, A.npz);
    } else {  // solid neighbour (Akinci 2012): pj.w = m_V_j, vj.w = -body density | -inf
        float cp = -(K.cps * pj.w) * g1;
        float fx = cp * rx, fy = cp * ry, fz = cp * rz;
        A.prx += fx; A.pry += fy; A.prz += fz;
        float body_rho = -vj.w;
        if (REACT && body_rho < 3.0e38f) {  // dynamic rigid: reaction, WCSPH.py:66-68
            float *a = reinterpret_cast<float *>(S.acc + j);
            float sc = -P.rho0 * rcp_ftz(body_rho);
            atomicAdd(a + 0, fx * sc);
            atomicAdd(a + 1, fy * sc);
            atomicAdd(a + 2, fz * sc);
        }
    }
}

// Fused force pass for uniform fluids: ONE 32-byte record gathered per neighbour (LDG.E.256) from the
// per-step copy fpv.  Because nothing reads posm / veld of OTHER particles here, FUSE_ADVECT lets the
// epilogue integrate the particle and clamp it to the walls in place (advect + enforce_boundary_3D
// (fluid), WCSPH.py:143-149, sph_base.py:149-179) -- one launch and one pass over the state less.
#ifndef FORCE_MIN_BLOCKS
#define FORCE_MIN_BLOCKS 6  // H100 sweep of 6-10 blocks/SM and batch 2 / 4: 6 x batch 4 is fastest (DESIGN.md 3.1)
#endif
#ifndef FORCE_BATCH
#define FORCE_BATCH 4
#endif
#ifndef FORCE_THREADS
#define FORCE_THREADS 128
#endif
// split_mode (sharded steps): 1 = only the particles inside the index ranges this rank sends to its neighbours
// (k_shard_info), 2 = only the others, 0 = all -- the halo exchange of the NEXT step starts as soon as the
// boundary particles are final and overlaps the interior.
static_assert(LIST_PAD % FORCE_BATCH == 0 && NBR_CAP % LIST_PAD == 0, "list padding must cover a force batch");

// Sharded boundary pass: the record of owned particle i, as it leaves this step, into the send staging of every side
// whose send range holds i -- slot (0, i - l0) / (1, i - r0), the slot k_shard_apply copies back from.
__device__ __forceinline__ void shard_stage_record(const DevParams &P, const DevArrays &S, int i, const float4 &p,
                                                   const float4 &v, const float4 &xo, const float4 &mi) {
    const int32_t *sd = S.sd;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
        const int b0 = side == 0 ? sd[SD_SEND_L0] : sd[SD_SEND_R0], b1 = side == 0 ? sd[SD_SEND_L1] : sd[SD_SEND_R1];
        if (i >= b0 && i < b1) {
            const int slot = i - b0;
            SPH_EMU_CHECK(slot < P.halo_cap);
            S.stage[side][0][slot] = p; S.stage[side][1][slot] = v; S.stage[side][2][slot] = xo; S.stage[side][3][slot] = mi;
        }
    }
}

// SHARD: the sharded steps' instantiation (send-range split, staging of the boundary particles); compile-time so
// that the single-GPU kernel keeps its register budget.
template <int B, int THREADS, bool FUSE_ADVECT, bool SHARD = false>
__global__ void __launch_bounds__(THREADS, FORCE_MIN_BLOCKS) k_force_packed(DevParams P, DevArrays S,
                                                                            int split_mode) {
    pdl_wait();
    auto one = [&](const int i) {
    float4 mi = S.misc[i];
    uint32_t fl = __float_as_uint(mi.z);
    if (!(fl & FLAG_FLUID)) {
        // a solid of a send range is staged too, unchanged: k_shard_apply copies the staging back over EVERY record
        // of the send ranges, and the neighbour's ghost copy comes from it (only the static-solid sequence splits)
        if (SHARD && FUSE_ADVECT && split_mode == 1) shard_stage_record(P, S, i, S.posm[i], S.veld[i], S.x0id[i], mi);
        return;
    }
    if (fl & FLAG_GHOST) return;
    float4 pi, vi;
    ldg256(S.fpv + 2 * (size_t)i, pi, vi);
    const float dpi = vi.w;
    PackedConst K;
    K.cohk = P.sigma / mi.x * P.fluid_m * P.k2_w;  // sigma / m_i * m_j
    K.cp = P.rho0 * P.fluid_mV;
    K.cps = P.rho0 * (dpi + mi.y * P.inv_rho0sq);
    ForceAcc A = {P.gx_, P.gy_, P.gz_, 0.f, 0.f, 0.f};
    const int cnt = S.nbr_cnt[i];
    if (cnt != NBR_OVERFLOW) {
        // 32-bit list slots (sph_create bounds NBR_CAP * npad below 2^32): one IADD + one IMAD.WIDE per load
        const uint32_t np = (uint32_t)S.npad;
        uint32_t slot = (uint32_t)i;
        for (int k0 = 0; k0 < cnt; k0 += B) {
            int j[B];  // the density pass padded the list to a multiple of LIST_PAD with i itself
            float4 pj[B], vj[B];
#pragma unroll
            for (int u = 0; u < B; ++u) j[u] = ldg_stream(S.nbr_list + (slot + (uint32_t)u * np));
#pragma unroll
            for (int u = 0; u < B; ++u) SPH_EMU_CHECK(k0 + u < NBR_CAP && j[u] >= 0 && j[u] < P.n);  // padded with i
#pragma unroll
            for (int u = 0; u < B; ++u) ldg256(S.fpv + 2 * (size_t)j[u], pj[u], vj[u]);
            slot += B * np;
            // all B gathers in flight before the first pair is evaluated: ptxas otherwise sinks three of
            // them below the arithmetic of pair 0, which then stalls on the first record with nothing
            // else outstanding.  (x | (y & 0)) with a zero it cannot see costs two LOP3 per batch.
            {
                uint32_t dep = 0u;
#pragma unroll
                for (int u = 1; u < B; ++u) dep ^= __float_as_uint(vj[u].w);
                pj[0].x = __uint_as_float(__float_as_uint(pj[0].x) | (dep & (uint32_t)P.opaque_zero));
            }
#pragma unroll
            for (int u = 0; u < B; ++u) {
                float rx = pi.x - pj[u].x, ry = pi.y - pj[u].y, rz = pi.z - pj[u].z;
                float r2 = rx * rx + ry * ry + rz * rz;
                force_pair_packed<!SHARD>(P, S, A, j[u], rx, ry, rz, r2, pj[u], vj[u], vi, dpi, K);
            }
        }
    } else {
        // full scan over the frozen copy (posm may already hold advected neighbours)
        for_all_neighbors<2>(P, S.fpv, S.cell_end, i, pi.x, pi.y, pi.z,
                             [&](int j, float rx, float ry, float rz, float r2, const float4 &pj) {
                                 force_pair_packed<!SHARD>(P, S, A, j, rx, ry, rz, r2, pj, __ldg(S.fpv + 2 * (size_t)j + 1),
                                                           vi, dpi, K);
                             });
    }
    float4 a = make_float4(A.npx + A.prx, A.npy + A.pry, A.npz + A.prz, 0.f);
    S.acc[i] = a;
    if (FUSE_ADVECT) {
        float4 p = make_float4(pi.x, pi.y, pi.z, P.fluid_mV);
        float4 v = make_float4(vi.x, vi.y, vi.z, S.veld[i].w);
        if (fl & FLAG_DYNAMIC) {
            v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
            p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
            wall_clamp(P, p, v);
        }
        if (SHARD && split_mode == 1) {
            // sharded boundary pass: the interior DENSITIES are still to come and read the positions of these
            // particles, so the advanced state goes to the send staging only (this IS the pack step; the halo
            // exchange starts right after this kernel) and k_shard_apply copies it back later
            shard_stage_record(P, S, i, p, v, S.x0id[i], mi);
        } else if (fl & FLAG_DYNAMIC) {
            S.posm[i] = p;
            S.veld[i] = v;
        }
    }
    };  // one particle
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    if (SHARD) {  // owned particles only, split into the send ranges and the rest
        const int32_t *sd = S.sd;
        if (i < sd[SD_OWN0] || i >= sd[SD_OWN1]) return;
        const bool boundary = (i >= sd[SD_SEND_L0] && i < sd[SD_SEND_L1]) || (i >= sd[SD_SEND_R0] && i < sd[SD_SEND_R1]);
        if (split_mode && (split_mode == 1) != boundary) return;
    }
    one(i);
}

// advect (WCSPH.py:143-149) for the dynamic SOLID particles only (companion of FUSE_ADVECT)
__global__ void k_advect_solids(DevParams P, DevArrays S) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.n_solid) return;
    int i = S.solid_slot[s];
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_DYNAMIC)) return;
    float4 p = S.posm[i], v = S.veld[i], a = S.acc[i];
    v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    S.posm[i] = p;
    S.veld[i] = v;
}

// =====================================================================================
// x-slab sharding with dynamic solids (sph_shard_configure_bodies, shard_bodies_sequence)
// =====================================================================================

// After k_rank_move (which also writes the slots of trash records) and a memset of the map to -1: the slot of every
// live record's solid id.  A second live record with the same id is a bookkeeping error (SPH_STATUS_SOLID_SLOT).
__global__ void k_shard_solid_slots(DevParams P, DevArrays S) {
    const int total = S.cell_end[P.C - 1];
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const int sid = __float_as_int(S.misc[t].w);
        if (sid < 0 || sid >= P.n_solid) continue;
        if (atomicMax(S.solid_slot + sid, t) != -1) atomicOr(S.status, SPH_STATUS_SOLID_SLOT);
    }
}

__device__ __forceinline__ bool shard_owned_index(const DevArrays &S, int i) {
    return i >= S.sd[SD_OWN0] && i < S.sd[SD_OWN1];  // false for -1; records of the owned layers are never ghosts
}

// The reactions of the fluid on the owned dynamic solids as a GATHER (the single engine scatters them from its force
// pass, which loses the fluid a neighbour owns across a cut), then advect (k_advect_solids).  One warp per solid j
// walks the 27 cells over the density pass's fpv records: the fluid of the owned layers and the first ghost layer,
// exactly the records whose fpv and pressure this step's density pass wrote.  Neighbour predicate and pair term are
// the force pass's, operand for operand (force_pair_packed, solid branch, with i the fluid and j the solid), so only
// the summation order differs from the single engine's float atomics.
__global__ void __launch_bounds__(128) k_shard_reactions(DevParams P, DevArrays S) {
    const int lane = threadIdx.x & 31;
    const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (s >= P.n_solid) return;  // warp-uniform
    const int j = S.solid_slot[s];
    if (!shard_owned_index(S, j)) return;
    if (!(__float_as_uint(S.misc[j].z) & FLAG_DYNAMIC)) return;
    const float4 pj = S.fpv[2 * (size_t)j], vj = S.fpv[2 * (size_t)j + 1];
    const float sc = -P.rho0 * rcp_ftz(-vj.w);  // -rho0 / body density
    const int d0 = S.sd[SD_DENS0], d1 = S.sd[SD_DENS1];
    int ci, cj, ck;
    cell_of(P, pj.x, pj.y, pj.z, ci, cj, ck);
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
                const float4 vi = __ldg(S.fpv + 2 * (size_t)i + 1);
                if (!(vi.w >= 0.0f)) continue;  // solid (fluid: p / rho^2 >= 0)
                const float4 pi = __ldg(S.fpv + 2 * (size_t)i);
                float rx = pi.x - pj.x, ry = pi.y - pj.y, rz = pi.z - pj.z;
                if (!(exact_r2(rx, ry, rz) < P.h2)) continue;  // the density pass's list predicate, symmetric in i, j
                float r2 = rx * rx + ry * ry + rz * rz;
                float wn, G;
                spline_pair(P, r2, wn, G);
                const float g1 = G * P.k1_grad;
                const float cps = P.rho0 * (vi.w + __ldg(&S.misc[i].y) * P.inv_rho0sq);
                float cp = -(cps * pj.w) * g1;
                ax += (cp * rx) * sc; ay += (cp * ry) * sc; az += (cp * rz) * sc;
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
    const float4 a = make_float4(P.gx_ + ax, P.gy_ + ay, P.gz_ + az, 0.f);
    float4 p = S.posm[j], v = S.veld[j];
    S.acc[j] = a;
    v.x += P.dt * a.x; v.y += P.dt * a.y; v.z += P.dt * a.z;
    p.x += P.dt * v.x; p.y += P.dt * v.y; p.z += P.dt * v.z;
    S.posm[j] = p;
    S.veld[j] = v;
}

// Shape matching across ranks.  The body solve must be the single engine's k_rigid bit for bit: its fp32 moments are
// summed in a fixed order over the solid ids (thread t of a 1024-thread CTA takes s = b0 + t, b0 + t + 1024, ..., then
// a fixed-order tree), and that rounding moves cm by ~1e-6 of the domain per step even in free fall -- a reduction in
// any other order or precision drifts from the single engine within a hundred steps and diverges after an impact.
// So every rank gathers the records of ALL body particles and repeats k_rigid's reduction on them.

// Offset of body b's particles in the gathered table (the bodies' particles in body order, then solid-id order).
__device__ __forceinline__ int shard_body_offset(const RigidBodyDev *bodies, int b) {
    int off = 0;
    for (int k = 0; k < b; ++k) off += bodies[k].solid_end - bodies[k].solid_begin;
    return off;
}

// Step 1 (one CTA per body): the clamps the earlier bodies' iterations apply first (k_rigid's pre_clamps), then this
// rank's entries of the table: rec[2k] = {x, m}, rec[2k + 1] = {x_0, 1} for the owned dynamic body particles, zeros
// (w = 0: not from this rank) for the others.
__global__ void k_shard_body_pack(DevParams P, DevArrays S, const RigidBodyDev *bodies, float4 *rec) {
    const int b = blockIdx.x, pre_clamps = b;
    const RigidBodyDev *B = bodies + b;
    const int b0 = B->solid_begin, off = shard_body_offset(bodies, b);
    for (int s = b0 + threadIdx.x; s < B->solid_end; s += blockDim.x) {
        float4 *r = rec + 2 * (size_t)(off + s - b0);
        const int i = S.solid_slot[s];
        if (!shard_owned_index(S, i) || !(__float_as_uint(S.misc[i].z) & FLAG_DYNAMIC)) {
            r[0] = make_float4(0.f, 0.f, 0.f, 0.f);
            r[1] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        float4 p = S.posm[i];
        if (pre_clamps > 0) {
            float4 v = S.veld[i];
            for (int k = 0; k < pre_clamps; ++k) wall_clamp(P, p, v);
            S.posm[i] = p;
            S.veld[i] = v;
        }
        const float4 x0 = S.x0id[i];
        r[0] = make_float4(p.x, p.y, p.z, P.m_V0 * S.veld[i].w);
        r[1] = make_float4(x0.x, x0.y, x0.z, 1.0f);
    }
}

// Step 2, after the all-gather of the tables (tables[world][n_rec][2]): one CTA of RIGID_THREADS per body runs k_rigid's
// mode-2 solve on the gathered records, each taken from the one rank that owns it -- the same operands in the same
// order, so cm and R equal the single engine's and are bit-identical on every rank.  They go to the body table; the
// owned body particles move to cm + R q and take this body's and the later bodies' clamps (k_rigid's post_clamps).
__global__ void __launch_bounds__(RIGID_THREADS) k_shard_body_solve(DevParams P, DevArrays S, RigidBodyDev *bodies,
                                                                    int n_bodies, const float4 *tables, int n_rec,
                                                                    int world) {
    __shared__ float red[32 * 16];
    __shared__ float s_R[9];
    const int body = blockIdx.x, post_clamps = n_bodies - body;
    RigidBodyDev *B = bodies + body;
    const int b0 = B->solid_begin, b1 = B->solid_end, off = shard_body_offset(bodies, body);
    const float r0 = B->rest_cm[0], r1 = B->rest_cm[1], r2 = B->rest_cm[2];
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int s = b0 + threadIdx.x; s < b1; s += blockDim.x) {
        const float4 *rec = nullptr;
        for (int r = 0; r < world && !rec; ++r) {
            const float4 *t = tables + 2 * ((size_t)r * n_rec + off + (s - b0));
            if (t[1].w != 0.0f) rec = t;
        }
        if (!rec) continue;  // not a dynamic particle (k_rigid skips it too)
        const float4 p = rec[0], x0 = rec[1];
        float mass = p.w;
        float q[3] = {x0.x - r0, x0.y - r1, x0.z - r2};
        float x[3] = {p.x, p.y, p.z};
        acc[0] += mass;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            acc[1 + r] += mass * x[r];
            acc[4 + r] += mass * q[r];
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[7 + 3 * r + c] += mass * x[r] * q[c];
        }
    }
    block_reduce<16>(acc, red);
    const float cmx = acc[1] / acc[0], cmy = acc[2] / acc[0], cmz = acc[3] / acc[0];
    if (threadIdx.x == 0) {
        const float cm[3] = {cmx, cmy, cmz};
        double Ad[9], Rd[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Ad[3 * r + c] = (double)acc[7 + 3 * r + c] - (double)cm[r] * (double)acc[4 + c];
        bool ok;
        polar_rotation_f64(Ad, Rd, ok);
        if (!ok) atomicOr(S.status, SPH_STATUS_BAD_POLAR);
        bool all_small = true;
        float Rf[9];
        for (int k = 0; k < 9; ++k) { Rf[k] = (float)Rd[k]; if (!(fabsf(Rf[k]) < 1e-6f)) all_small = false; }
        if (all_small) { for (int k = 0; k < 9; ++k) Rf[k] = (k % 4 == 0) ? 1.0f : 0.0f; }
        for (int k = 0; k < 9; ++k) { s_R[k] = Rf[k]; B->R[k] = Rf[k]; }
        B->cm[0] = cmx; B->cm[1] = cmy; B->cm[2] = cmz;
    }
    __syncthreads();
    for (int s = b0 + threadIdx.x; s < b1; s += blockDim.x) {
        const int i = S.solid_slot[s];
        if (!shard_owned_index(S, i)) continue;
        uint32_t fl = __float_as_uint(S.misc[i].z);
        if (!(fl & FLAG_DYNAMIC)) continue;
        float4 p = S.posm[i], x0 = S.x0id[i];
        float q0 = x0.x - r0, q1 = x0.y - r1, q2 = x0.z - r2;
        float gx = cmx + (s_R[0] * q0 + s_R[1] * q1 + s_R[2] * q2);
        float gy = cmy + (s_R[3] * q0 + s_R[4] * q1 + s_R[5] * q2);
        float gz = cmz + (s_R[6] * q0 + s_R[7] * q1 + s_R[8] * q2);
        p.x += (gx - p.x) * 1.0f; p.y += (gy - p.y) * 1.0f; p.z += (gz - p.z) * 1.0f;
        if (post_clamps > 0) {
            float4 v = S.veld[i];
            for (int r = 0; r < post_clamps; ++r) wall_clamp(P, p, v);
            S.veld[i] = v;
        }
        S.posm[i] = p;
    }
}

// =====================================================================================
// sph_shard_dump: x and v of one object's owned records, compacted in sorted order
// =====================================================================================
// Three passes over the owned index range [own0, own1) of the last sort, in tiles of DUMP_TILE consecutive records
// (one block each, DUMP_ROUNDS rounds of DUMP_THREADS records): count the kept records per tile (ballot + popc), one
// block scans the tile counts, and the tiles scatter their records to the scanned row offsets.  Within a tile the
// rows follow the rounds, then the warps, then the lanes, i.e. the index order: the compaction keeps the sorted
// order and is the same on every run.
constexpr int DUMP_THREADS = 256;
constexpr int DUMP_ROUNDS = 4;
constexpr int DUMP_TILE = DUMP_THREADS * DUMP_ROUNDS;
constexpr int DUMP_WARPS = DUMP_THREADS / 32;

// a record of the object that this rank owns (the set ShardedSimulation.owned_tensors takes)
__device__ __forceinline__ bool dump_keep(const DevArrays &S, int i, int32_t object_id) {
    return __float_as_int(S.x0id[i].w) == object_id && !(__float_as_uint(S.misc[i].z) & FLAG_GHOST);
}

// counts[b] = kept records of tile b
__global__ void __launch_bounds__(DUMP_THREADS) k_dump_count(DevArrays S, int own0, int own1, int32_t object_id,
                                                             int32_t *counts) {
    __shared__ int warp_rows[DUMP_WARPS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int base = own0 + blockIdx.x * DUMP_TILE;
    int rows = 0;  // this warp's kept records (the same in every lane)
    for (int k = 0; k < DUMP_ROUNDS; ++k) {
        const int i = base + k * DUMP_THREADS + threadIdx.x;
        rows += __popc(__ballot_sync(0xffffffffu, i < own1 && dump_keep(S, i, object_id)));
    }
    if (lane == 0) warp_rows[w] = rows;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int q = 0; q < DUMP_WARPS; ++q) t += warp_rows[q];
        counts[blockIdx.x] = t;
    }
}

// ONE block: counts[0, n_tiles) -> exclusive prefix sums in place, counts[n_tiles] = the total
__global__ void __launch_bounds__(DUMP_THREADS) k_dump_scan(int32_t *counts, int n_tiles) {
    __shared__ int warp_rows[DUMP_WARPS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int carry = 0;  // rows of the chunks before this one (the same in every thread)
    for (int c0 = 0; c0 < n_tiles; c0 += DUMP_THREADS) {
        const int b = c0 + threadIdx.x;
        const int mine = b < n_tiles ? counts[b] : 0;
        int incl = mine;
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) warp_rows[w] = incl;
        __syncthreads();
        int before = carry, chunk = 0;
        for (int q = 0; q < DUMP_WARPS; ++q) {
            before += q < w ? warp_rows[q] : 0;
            chunk += warp_rows[q];
        }
        __syncthreads();  // every thread has read warp_rows before the next chunk writes it
        if (b < n_tiles) counts[b] = before + incl - mine;
        carry += chunk;
    }
    if (threadIdx.x == 0) counts[n_tiles] = carry;
}

// x[3 r..3 r + 2], v[...] of the kept records, r = the record's row (offsets: k_dump_scan's prefix sums)
__global__ void __launch_bounds__(DUMP_THREADS) k_dump_scatter(DevArrays S, int own0, int own1, int32_t object_id,
                                                               const int32_t *offsets, float *x, float *v) {
    __shared__ int warp_rows[DUMP_ROUNDS][DUMP_WARPS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int base = own0 + blockIdx.x * DUMP_TILE;
    unsigned keep[DUMP_ROUNDS];
#pragma unroll
    for (int k = 0; k < DUMP_ROUNDS; ++k) {
        const int i = base + k * DUMP_THREADS + threadIdx.x;
        keep[k] = __ballot_sync(0xffffffffu, i < own1 && dump_keep(S, i, object_id));
        if (lane == 0) warp_rows[k][w] = __popc(keep[k]);
    }
    __syncthreads();
    int row = offsets[blockIdx.x];  // first row of this round
#pragma unroll
    for (int k = 0; k < DUMP_ROUNDS; ++k) {
        int r = row + __popc(keep[k] & ((1u << lane) - 1u));
        for (int q = 0; q < DUMP_WARPS; ++q) {
            r += q < w ? warp_rows[k][q] : 0;
            row += warp_rows[k][q];
        }
        if ((keep[k] >> lane) & 1u) {
            const int i = base + k * DUMP_THREADS + threadIdx.x;
            const float4 a = S.posm[i], b = S.veld[i];
            x[3 * (size_t)r] = a.x; x[3 * (size_t)r + 1] = a.y; x[3 * (size_t)r + 2] = a.z;
            v[3 * (size_t)r] = b.x; v[3 * (size_t)r + 1] = b.y; v[3 * (size_t)r + 2] = b.z;
        }
    }
}

// Diagnostics: neighbour-list statistics of the last density pass -> out[4] = {max count, particles in
// overflow (full-scan fallback), total pairs, particles with a list}.  out must be zeroed by the caller.
__global__ void k_neighbor_stats(DevParams P, DevArrays S, int32_t *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    if (P.slab_on && i >= S.sd[SD_N_LIVE]) return;
    uint32_t fl = __float_as_uint(S.misc[i].z);
    if (!(fl & FLAG_FLUID)) return;
    int c = S.nbr_cnt[i];
    if (c == NBR_OVERFLOW) { atomicAdd(out + 1, 1); c = NBR_CAP; }
    atomicMax(out + 0, c);
    atomicAdd(out + 2, c);
    atomicAdd(out + 3, 1);
}
