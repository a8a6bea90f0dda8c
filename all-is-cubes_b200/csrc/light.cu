// light.cu — host side of the secondary path (SURVEY §8(a) L1-L4): the static light-ray chart
// (space/light/chart/generator.rs), the per-block derived table, and the batched relaxation driver
// replacing LightStorage::update_light_from_queue / apply_light_update / fast_evaluate_light /
// modified_cube_needs_update (space/light/updater.rs) and Mutation::evaluate_light (space.rs:1496-1527).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include <cub/device/device_scan.cuh>

#include "internal.h"
#include "light_kernel.cuh"

using namespace aicb;
using namespace aicb_light;

// ---------------------------------------------------------------------------------------------
// chart generation (generator.rs:49-215) — host, once per context
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int CHAIN_WALK_BLOCKS_PER_SM = 6;   // 4 warps, 80 registers, 26 KB of shared memory each
// Cubes within 16 priority levels of the round's maximum are relaxed together: far fewer rounds than strict
// level-by-level relaxation (few cubes per round leave the GPU idle) for 8 % more updates.
constexpr uint32_t PRIORITY_BAND = 16;

struct TreeNode {
    int8_t cube[3];
    int children[6];
    float weight[6];
};

// scale_to_integer_step (raycast.rs:797-819) for s = 0.5
double stis_half(double ds) {
    if (ds == 0.0) return INFINITY;
    return (1.0 - 0.5) / std::fabs(ds);  // rem_euclid(+-0.5, 1) == 0.5 either way
}

std::vector<LightChartNode> build_chart() {
    std::vector<TreeNode> pool;
    pool.push_back(TreeNode{{0, 0, 0}, {-1, -1, -1, -1, -1, -1}, {0, 0, 0, 0, 0, 0}});
    const int R = 5;  // RAY_DIRECTION_STEP
    for (int x = -R; x <= R; x++)
        for (int y = -R; y <= R; y++)
            for (int z = -R; z <= R; z++) {
                if (!(std::abs(x) == R || std::abs(y) == R || std::abs(z) == R)) continue;
                const float fx = (float)x, fy = (float)y, fz = (float)z;
                const float len = std::sqrt(fx * fx + fy * fy + fz * fz);
                const float d[3] = {fx / len, fy / len, fz / len};  // Vector3D::normalize
                float cos6[6];
                for (int f = 0; f < 6; f++) {
                    float u[3] = {0, 0, 0};
                    u[f % 3] = (f < 3) ? -1.0f : 1.0f;
                    const float dot = u[0] * d[0] + u[1] * d[1] + u[2] * d[2];
                    cos6[f] = std::fmax(dot, 0.0f);
                }
                // ray_to_steps (generator.rs:100-113): Ray::new([0.5;3], direction).cast(), t <= 127.
                // Unbounded Raycaster (raycast.rs:577-626) from the cube (0,0,0).
                const double dd[3] = {(double)d[0], (double)d[1], (double)d[2]};
                int step[3];
                double t_delta[3], t_max[3];
                for (int a = 0; a < 3; a++) {
                    step[a] = dd[a] == 0.0 ? 0 : (dd[a] < 0.0 ? -1 : 1);
                    t_delta[a] = 1.0 / std::fabs(dd[a]);
                    t_max[a] = stis_half(dd[a]);
                }
                int cube[3] = {0, 0, 0};
                for (int f = 0; f < 6; f++) pool[0].weight[f] += cos6[f];  // the root is on every path
                int cur = 0;
                for (;;) {
                    int axis;
                    if (t_max[0] < t_max[1]) axis = (t_max[0] < t_max[2]) ? 0 : 2;
                    else axis = (t_max[1] < t_max[2]) ? 1 : 2;
                    const double t = t_max[axis];
                    cube[axis] += step[axis];
                    t_max[axis] += t_delta[axis];
                    if (!(t <= 127.0)) break;
                    const int dir = step[axis] > 0 ? 3 + axis : axis;  // Face::from_adjacency(previous, this)
                    int child = pool[cur].children[dir];
                    if (child < 0) {
                        child = (int)pool.size();
                        pool[cur].children[dir] = child;
                        pool.push_back(TreeNode{{(int8_t)cube[0], (int8_t)cube[1], (int8_t)cube[2]}, {-1, -1, -1, -1, -1, -1}, {0, 0, 0, 0, 0, 0}});
                    }
                    cur = child;
                    for (int f = 0; f < 6; f++) pool[cur].weight[f] += cos6[f];
                }
            }
    std::vector<LightChartNode> flat(pool.size());
    for (size_t i = 0; i < pool.size(); i++)
        for (int f = 0; f < 6; f++) {
            flat[i].w[f] = pool[i].weight[f];
            flat[i].child[f] = pool[i].children[f] < 0 ? 0u : (uint32_t)pool[i].children[f];
        }
    return flat;
}

// The chart in depth-first preorder, as the lockstep walk (light_kernel.cuh) steps through it: children in Face6
// order (the order walk_ray_tree recurses in, updater.rs:500), each node with its depth, its cube relative to the
// origin, the direction of the step from its parent and the index one past its last descendant.
std::vector<LightNodePre> build_chart_preorder(const std::vector<LightChartNode> &flat, std::vector<uint32_t> *flat_index = nullptr) {
    std::vector<LightNodePre> pre;
    pre.reserve(flat.size());
    struct Item { uint32_t node; int8_t rel[3]; uint8_t depth; uint8_t dir; uint32_t slot; uint8_t next_child; };
    std::vector<Item> stack;
    stack.push_back(Item{0, {0, 0, 0}, 0, 0, 0, 0});
    while (!stack.empty()) {
        Item &it = stack.back();
        if (it.next_child == 0) {   // first visit: emit the node
            it.slot = (uint32_t)pre.size();
            LightNodePre n;
            std::memcpy(n.w, flat[it.node].w, sizeof n.w);
            n.rel[0] = it.rel[0]; n.rel[1] = it.rel[1]; n.rel[2] = it.rel[2];
            n.depth = it.depth;
            n.end_dir = (uint32_t)it.dir << 29;
            pre.push_back(n);
            if (flat_index) flat_index->push_back(it.node);
        }
        int f = it.next_child;
        while (f < 6 && flat[it.node].child[f] == 0) f++;
        if (f < 6) {
            it.next_child = (uint8_t)(f + 1);
            Item c;
            c.node = flat[it.node].child[f];
            c.rel[0] = it.rel[0]; c.rel[1] = it.rel[1]; c.rel[2] = it.rel[2];
            c.rel[f % 3] = (int8_t)(c.rel[f % 3] + ((f < 3) ? -1 : 1));
            c.depth = (uint8_t)(it.depth + 1);
            c.dir = (uint8_t)f;
            c.slot = 0;
            c.next_child = 0;
            stack.push_back(c);   // (invalidates `it`)
        } else {
            pre[it.slot].end_dir |= (uint32_t)pre.size();
            stack.pop_back();
        }
    }
    return pre;
}

const std::vector<LightNodePre> &chart_preorder_host() {
    static const std::vector<LightNodePre> pre = build_chart_preorder(build_chart());
    return pre;
}

// The chart as chains (light_kernel.cuh: LightChain): maximal single-child paths of the preorder chart, numbered
// breadth first; the Euler tour of the chain tree is the depth-first order the terms of a walk are added in.
struct ChainTables {
    std::vector<LightChain> chains;
    std::vector<uchar4> node_rel;
    std::vector<uint16_t> euler;
};
const ChainTables &chain_tables_host() {
    static const ChainTables tables = [] {
        const std::vector<LightNodePre> &pre = chart_preorder_host();
        const uint32_t n = (uint32_t)pre.size();
        auto end_of = [&](uint32_t i) { return pre[i].end_dir & 0x1fffffffu; };
        auto children_of = [&](uint32_t i) {
            std::vector<uint32_t> c;
            for (uint32_t k = i + 1; k < end_of(i); k = end_of(k)) c.push_back(k);
            return c;
        };
        ChainTables t;
        t.node_rel.resize(n);
        for (uint32_t i = 0; i < n; i++)
            t.node_rel[i] = make_uchar4((uint8_t)pre[i].rel[0], (uint8_t)pre[i].rel[1], (uint8_t)pre[i].rel[2], (uint8_t)(pre[i].end_dir >> 29));
        std::vector<uint32_t> start;           // chain -> first node
        std::vector<uint16_t> parent_branch;
        start.push_back(0);
        parent_branch.push_back(0xffff);
        uint16_t n_branches = 0;
        for (size_t c = 0; c < start.size(); c++) {
            LightChain ch;
            std::memset(&ch, 0, sizeof ch);
            std::memcpy(ch.w, pre[start[c]].w, sizeof ch.w);
            ch.first_node = start[c];
            uint32_t e = start[c];
            std::vector<uint32_t> kids = children_of(e);
            while (kids.size() == 1) { e = kids[0]; kids = children_of(e); }
            ch.length = (uint16_t)(e - start[c] + 1);
            ch.n_children = (uint8_t)kids.size();
            ch.parent_branch = parent_branch[c];
            ch.branch = kids.empty() ? (uint16_t)0xffff : n_branches++;
            ch.first_child = (uint32_t)start.size();
            for (uint32_t k : kids) { start.push_back(k); parent_branch.push_back(ch.branch); }
            t.chains.push_back(ch);
        }
        // Euler tour (iterative): enter(c), children in order, exit(c)
        struct It { uint32_t c; uint32_t next; };
        std::vector<It> stack;
        stack.push_back(It{0, 0});
        t.euler.push_back(0);
        while (!stack.empty()) {
            It &it = stack.back();
            const LightChain &ch = t.chains[it.c];
            if (it.next < ch.n_children) {
                const uint32_t k = ch.first_child + it.next++;
                t.euler.push_back((uint16_t)k);
                stack.push_back(It{k, 0});
            } else {
                t.euler.push_back((uint16_t)(it.c | 0x8000u));
                stack.pop_back();
            }
        }
        return t;
    }();
    return tables;
}

// The chart's tables on the context's device; the context takes them once every one is uploaded.
aicb_status ensure_chart(aicb_ctx *ctx) {
    if (ctx->light_chart.pre) return AICB_OK;
    const ChainTables &t = chain_tables_host();
    if (t.chains.size() > (size_t)LIGHT_MAX_CHAINS || t.chains.size() >= 0x8000u)
        return aicb_fail(AICB_ERR_INVALID, "light chart has more chains than the walk's shared arrays hold");
    size_t branches = 0;
    for (const LightChain &c : t.chains) branches += c.n_children ? 1 : 0;
    if (branches > (size_t)LIGHT_MAX_BRANCHES) return aicb_fail(AICB_ERR_INVALID, "light chart has more branching chains than expected");
    LightChart c;
    TRY(c.chains.upload(t.chains));
    TRY(c.node_rel.upload(t.node_rel));
    TRY(c.euler.upload(t.euler));
    c.walk_blocks = (uint32_t)ctx->num_sms * CHAIN_WALK_BLOCKS_PER_SM;
    // one set of term slots per resident warp of the chain walk
    TRY(c.term_scratch.ensure((size_t)c.walk_blocks * 4 * LIGHT_WARP_SCRATCH_F4 * sizeof(float4)));
    const std::vector<LightNodePre> &pre = chart_preorder_host();
    TRY(c.pre.upload(pre));
    c.nodes = (uint32_t)pre.size();
    c.n_chains = (uint32_t)t.chains.size();
    c.n_euler = (uint32_t)t.euler.size();
    ctx->light_chart = std::move(c);
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
// The queue: one priority byte per cube (0 = not queued) and, per LIGHT_TILE cubes, an upper bound of the tile's
// highest byte (raised with every insert, recomputed by whoever scans the tile).  Finding the round's priority reads
// the tile bounds only; gathering reads only the tiles that can hold a cube of the round.
__global__ void __launch_bounds__(256) k_tile_rebuild(const LightParams P, uint32_t n_tiles) {
    __shared__ uint32_t s_max[8];
    const uint32_t n_words = (P.volume + 3) / 4;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t w = tile * (LIGHT_TILE / 4) + threadIdx.x;
        const uint32_t v = w < n_words ? ((const uint32_t *)P.pending)[w] : 0u;
        uint32_t m = max(max(v & 255u, (v >> 8) & 255u), max((v >> 16) & 255u, v >> 24));
        for (int off = 16; off > 0; off >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, off));
        if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t t = 0;
            for (int i = 0; i < 8; i++) t = max(t, s_max[i]);
            P.tile_max[tile] = t;
        }
        __syncthreads();
    }
}

__global__ void k_find_max(const LightParams P, uint32_t n_tiles) {
    uint32_t m = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_tiles; i += gridDim.x * blockDim.x) m = max(m, P.tile_max[i]);
    for (int off = 16; off > 0; off >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&P.counters->priority, m);
}

// A round whose priority is already <= epsilon does nothing.
// One block per tile: the cubes of a tile reach the list in index order (block-wide scan), so 32 consecutive list
// entries are neighbours along z — what the lockstep walk wants.
// Thread -> word of the tile whose cubes a gathering thread lists.  With a power-of-two z extent the tile is a few whole
// z-rows, and the threads are laid out so that 8 consecutive threads (32 cubes: one warp of the lockstep walk) cover a
// 4 x 8 patch of (y, z) instead of 32 cubes in a line: neighbours in two directions share more of their chart walk.
__device__ __forceinline__ uint32_t list_word_of_thread(const LightParams &P) {
    uint32_t wl = threadIdx.x;
    const uint32_t nz = (uint32_t)P.scene.size[2];
    if (nz >= 8 && nz <= 256 && (nz & (nz - 1)) == 0) {
        const uint32_t wpr = nz / 4, q = threadIdx.x >> 3, within = threadIdx.x & 7;
        const uint32_t row_group = q / (wpr / 2), pz = q % (wpr / 2);
        wl = (row_group * 4 + (within >> 1)) * wpr + pz * 2 + (within & 1);
    }
    return wl;
}

__global__ void __launch_bounds__(256) k_gather(const LightParams P, uint32_t n_tiles) {
    __shared__ uint32_t s_part[8], s_max[8], s_base;
    const uint32_t prio = P.counters->priority;
    if (prio <= P.epsilon_priority) return;
    const uint32_t n_words = (P.volume + 3) / 4;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t wl = list_word_of_thread(P);
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t tm = P.tile_max[tile];
        if (tm <= P.epsilon_priority || tm + PRIORITY_BAND < prio) continue;   // (block-uniform)
        const uint32_t w = tile * (LIGHT_TILE / 4) + wl;
        uint32_t v = w < n_words ? ((uint32_t *)P.pending)[w] : 0u;
        uint32_t sel = 0, cnt = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            const uint32_t p = (v >> (8 * k)) & 255u;
            if (p > P.epsilon_priority && p + PRIORITY_BAND >= prio && w * 4 + k < P.volume) { sel |= 1u << k; cnt++; }
        }
        // exclusive scan of cnt over the block
        uint32_t inc = cnt;
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
            if ((int)lane >= off) inc += t;
        }
        if (lane == 31) s_part[wid] = inc;
        // what stays queued in this tile
        uint32_t rest = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) if (!(sel & (1u << k))) rest = max(rest, (v >> (8 * k)) & 255u);
        for (int off = 16; off > 0; off >>= 1) rest = max(rest, __shfl_down_sync(0xffffffffu, rest, off));
        if (lane == 0) s_max[wid] = rest;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t total = 0, m = 0;
            for (int i = 0; i < 8; i++) { const uint32_t c = s_part[i]; s_part[i] = total; total += c; m = max(m, s_max[i]); }
            s_base = total ? atomicAdd(&P.counters->gathered, total) : 0u;
            P.tile_max[tile] = m;
        }
        __syncthreads();
        if (cnt) {
            uint32_t at = s_base + s_part[wid] + inc - cnt;
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)
                if (sel & (1u << k)) { P.list[at++] = w * 4 + k; v &= ~(255u << (8 * k)); }
            ((uint32_t *)P.pending)[w] = v;
        }
        __syncthreads();
    }
}

// compute_light / the dependency re-queue with the chain walk (light_kernel.cuh: compute_light_chains): one warp per
// cube, cubes handed out by a counter.  k_walk_chains<false> writes new_light for the round's list (or explicit
// cubes); a cube one of whose chains needs more than LIGHT_CHAIN_K terms goes to the overflow list and is computed by
// the lockstep walk (k_compute_overflow).  k_walk_chains<true> re-queues the dependencies of the entries of `changed`.
// RECORD (k_walk_chains_record): the compute form for explicit cubes that also logs every cube's rays and which cubes
// overflowed.
template <bool MARK, bool RECORD>
__device__ __forceinline__ void walk_chains(const LightParams &P, uint32_t n, const int32_t *explicit_cubes,
                                            const LightRayLog &log) {
    __shared__ float s_lut[256];
    __shared__ ChainShared s_sh[4];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    ChainShared &sh = s_sh[wib];
    float4 *terms = P.term_scratch + (size_t)(blockIdx.x * 4 + wib) * LIGHT_WARP_SCRATCH_F4;
    if (!explicit_cubes) n = MARK ? P.counters->changed : P.counters->gathered;
    unsigned long long total_visits = 0;
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(MARK ? &P.counters->mark_work : &P.counters->compute_work, 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= n) break;
        const uint32_t i = MARK ? P.changed[item] : item;   // position in the round's list
        int x, y, z;
        if (explicit_cubes) { x = explicit_cubes[3 * i]; y = explicit_cubes[3 * i + 1]; z = explicit_cubes[3 * i + 2]; }
        else cube_of(P.scene, P.list[i], x, y, z);
        const uint32_t prio = MARK ? (uint32_t)P.diff[i] / 2u + 1u : 0u;
        uint32_t visits = 0;
        bool overflowed = false;
        const uint32_t nv = compute_light_chains<MARK, RECORD>(P, s_lut, sh, terms, x, y, z, prio, &visits, &overflowed,
                                                               log, i);
        if (!MARK && lane == 0) {
            if (overflowed) P.overflow[atomicAdd(P.overflow_count, 1u)] = i;
            else P.new_light[i] = nv;
            if (RECORD) log.lockstep[i] = overflowed ? 1 : 0;
        }
        total_visits += visits;
    }
    if (!MARK && lane == 0 && total_visits) atomicAdd(&P.counters->node_visits, total_visits);
}
template <bool MARK>
__global__ void __launch_bounds__(128, CHAIN_WALK_BLOCKS_PER_SM) k_walk_chains(const LightParams P, uint32_t n, const int32_t *explicit_cubes) {
    walk_chains<MARK, false>(P, n, explicit_cubes, LightRayLog());
}
__global__ void __launch_bounds__(128) k_walk_chains_record(const LightParams P, uint32_t n, const int32_t *explicit_cubes,
                                                            const LightRayLog log) {
    walk_chains<false, true>(P, n, explicit_cubes, log);
}

// 8 CTAs of 4 warps per SM (64 registers; the records requested ahead spill to L1-resident local memory): the walk is
// latency bound, so 32 resident warps serve it better than the 20 that 94 registers would allow.
constexpr int LOCKSTEP_MIN_BLOCKS = 8;

// the cubes the chain walk could not hold (*overflow_count entries of `overflow`), by the lockstep walk; RECORD
// (k_compute_overflow_record) also logs their rays
template <bool RECORD>
__device__ __forceinline__ void compute_overflow(const LightParams &P, const int32_t *explicit_cubes, const LightRayLog &log) {
    __shared__ float s_lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    const uint32_t n = *P.overflow_count;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    unsigned long long total_visits = 0;
    for (uint32_t base = warp * 32u; base < n; base += n_warps * 32u) {
        const bool active = base + lane < n;
        const uint32_t i = active ? P.overflow[base + lane] : 0u;
        int x = 0, y = 0, z = 0;
        if (active) {
            if (explicit_cubes) { x = explicit_cubes[3 * i]; y = explicit_cubes[3 * i + 1]; z = explicit_cubes[3 * i + 2]; }
            else cube_of(P.scene, P.list[i], x, y, z);
        }
        uint32_t visits = 0;
        const uint32_t nv = compute_light_lockstep<RECORD>(P, s_lut, active, x, y, z, &visits, log, i);
        if (active) P.new_light[i] = nv;
        total_visits += visits;
    }
    for (int off = 16; off > 0; off >>= 1) total_visits += __shfl_down_sync(0xffffffffu, total_visits, off);
    if (lane == 0 && total_visits) atomicAdd(&P.counters->node_visits, total_visits);
}
__global__ void __launch_bounds__(128, LOCKSTEP_MIN_BLOCKS) k_compute_overflow(const LightParams P, const int32_t *explicit_cubes) {
    compute_overflow<false>(P, explicit_cubes, LightRayLog());
}
__global__ void __launch_bounds__(128) k_compute_overflow_record(const LightParams P, const int32_t *explicit_cubes,
                                                                 const LightRayLog log) {
    compute_overflow<true>(P, explicit_cubes, log);
}

// A texel of device 0's light volume was written: its 32-cube segment goes to the other replicas (k_push).
__device__ __forceinline__ void mark_dirty(const LightParams &P, uint32_t idx) {
    atomicOr(P.dirty + idx / 1024u, 1u << ((idx / 32u) & 31u));
}

// A light call wrote the cube's texel: it enters the set of changed cubes (SpaceChange::CubeLight).
__device__ __forceinline__ void mark_changed(const LightParams &P, uint32_t idx) {
    atomicOr(P.changes + idx / 32u, 1u << (idx & 31u));
}

// apply_light_update (updater.rs:295-363) minus the dependency re-queue (k_walk_chains<true>).  Every stored value and
// every guess written into an Uninitialized neighbour enters the set of changed cubes (updater.rs:313-317, 335-338).
// GROUP: device 0 of a group also marks every texel it writes dirty.
template <bool GROUP>
__global__ void k_apply(const LightParams P) {
    const uint32_t n = P.counters->gathered;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t idx = P.list[i];
    uint32_t *light = const_cast<uint32_t *>(P.scene.light);
    const uint32_t old = light[idx], nv = P.new_light[i];
    const int d = difference_priority(nv, old);
    P.diff[i] = (uint8_t)d;
    atomicAdd(&P.counters->updates, 1u);
    if (d > 0) {
        light[idx] = nv;
        mark_changed(P, idx);
        if (GROUP) mark_dirty(P, idx);
        atomicMax(&P.counters->max_diff, (uint32_t)d);
        int x, y, z;
        cube_of(P.scene, idx, x, y, z);
        const float *lut = P.scene.tables;
#pragma unroll
        for (int f = 0; f < 6; f++) {
            const int s = (f < 3) ? -1 : 1, a = f % 3;
            uint32_t nidx;
            if (!cube_index(P.scene, x + (a == 0 ? s : 0), y + (a == 1 ? s : 0), z + (a == 2 ? s : 0), &nidx)) continue;
            const uint32_t nl = light[nidx];
            if ((nl >> 24) != 0) continue;            // only LightStatus::Uninitialized neighbours
            if (nl == nv) continue;
            if (__ldg(&P.blocks[block_id_at(P.scene, nidx)].flags) & LB_ALL_OPAQUE) continue;
            // PackedLight::guess(new.value()): re-quantise the decoded value, status Uninitialized
            const uint32_t g = scalar_in_t(lut, lut[nv & 255]) | (scalar_in_t(lut, lut[(nv >> 8) & 255]) << 8) | (scalar_in_t(lut, lut[(nv >> 16) & 255]) << 16);
            const uint32_t prev = atomicCAS(&light[nidx], nl, g);
            if (prev == nl) {
                mark_changed(P, nidx);
                if (GROUP) mark_dirty(P, nidx);
            }
        }
    }
    }
}

// The push of a group's round: every 32-cube segment of device 0's light volume that k_apply wrote (one 128-byte
// line) is stored into the other replicas' volumes over NVLink, and its dirty bit cleared.  It runs after k_apply, so
// it stores the final values even where two guesses raced for one neighbour.  One warp per word of dirty bits.
__global__ void __launch_bounds__(256) k_push(const LightParams P, uint32_t *const *targets, uint32_t n_targets) {
    const uint32_t n_words = (P.volume + 1023u) / 1024u;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t w = warp; w < n_words; w += n_warps) {
        uint32_t bits = __shfl_sync(0xffffffffu, lane == 0 ? P.dirty[w] : 0u, 0);
        if (!bits) continue;
        if (lane == 0) P.dirty[w] = 0u;
        while (bits) {
            const uint32_t idx = (w * 32u + (uint32_t)(__ffs(bits) - 1)) * 32u + lane;
            bits &= bits - 1u;
            if (idx < P.volume) {
                const uint32_t v = P.scene.light[idx];
                for (uint32_t t = 0; t < n_targets; t++) targets[t][idx] = v;
            }
        }
    }
}

// apply_light_update re-queues a cube's dependencies only when its packed difference exceeds 1 (updater.rs:355-360).
// The entries of the round's list that did are compacted (in list order within a block of 256) so that
// k_walk_chains<true> walks the chart only for cubes that need it.
__global__ void __launch_bounds__(256) k_compact_changed(const LightParams P) {
    __shared__ uint32_t s_part[8], s_base;
    const uint32_t n = P.counters->gathered;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t base = blockIdx.x * 256u; base < n; base += gridDim.x * 256u) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t keep = (i < n && P.diff[i] > 1) ? 1u : 0u;
        uint32_t inc = keep;
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
            if ((int)lane >= off) inc += t;
        }
        if (lane == 31) s_part[wid] = inc;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t total = 0;
            for (int k = 0; k < 8; k++) { const uint32_t c = s_part[k]; s_part[k] = total; total += c; }
            s_base = total ? atomicAdd(&P.counters->changed, total) : 0u;
        }
        __syncthreads();
        if (keep) P.changed[s_base + s_part[wid] + inc - 1] = i;
        __syncthreads();
    }
}

// fast_evaluate_light (updater.rs:537-582): one thread per (x, z) column, top down.  The reference announces none of
// these writes (its TODO for EveryBlock); a texel whose value changes enters the set of changed cubes all the same.
__global__ void k_fast_evaluate(const LightParams P) {
    const DeviceScene &S = P.scene;
    const uint32_t col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= (uint32_t)S.size[0] * (uint32_t)S.size[2]) return;
    const int x = (int)(col / (uint32_t)S.size[2]) + S.lo[0], z = (int)(col % (uint32_t)S.size[2]) + S.lo[2];
    uint32_t *light = const_cast<uint32_t *>(S.light);
    bool covered = false;
    for (int y = S.lo[1] + S.size[1] - 1; y >= S.lo[1]; y--) {
        uint32_t idx;
        cube_index(S, x, y, z, &idx);
        const uint32_t fl = __ldg(&P.blocks[block_id_at(S, idx)].flags);
        uint32_t value;
        uint8_t pend = 0;
        if ((fl & LB_ALL_OPAQUE) && !(fl & LB_EMISSIVE)) {
            covered = true;
            value = TX_OPAQUE;
        } else {
            bool any = (fl & LB_VISIBLE) != 0;
            if (!any) {
                any = (flags_at(P, x - 1, y, z) | flags_at(P, x + 1, y, z) | flags_at(P, x, y - 1, z) | flags_at(P, x, y + 1, z) |
                       flags_at(P, x, y, z - 1) | flags_at(P, x, y, z + 1)) & LB_VISIBLE;
            }
            if (any) {
                pend = PRIO_ESTIMATED;
                value = covered ? TX_UNINIT : S.sky_faces[4];  // block_sky.in_direction(PY)
            } else {
                value = TX_NO_RAYS;
            }
        }
        if (light[idx] != value) mark_changed(P, idx);
        light[idx] = value;
        P.pending[idx] = pend;
    }
}

// modified_cube_needs_update (updater.rs:135-173) for a cube that holds block `id`: a block opaque for light stores
// OPAQUE (a changed cube even if it already was, updater.rs:153-161) and cancels the cube's queued update, any other
// block queues the cube at NEWLY_VISIBLE; then the face neighbours whose own face toward the cube is not opaque are
// queued.  Only `queue` (device 0 of a group) touches the queue and the set.  Threads may apply it to any set of cubes
// at once, reading the cells as they are after every edit: no two threads write one pending byte with different
// values, since a cube opaque for light is opaque on every face, so no neighbour queues it, and every other write
// stores NEWLY_VISIBLE.
__device__ __forceinline__ void modified_cube(const LightParams &P, uint32_t idx, uint32_t id, uint32_t queue) {
    const uint32_t fl = __ldg(&P.blocks[id].flags);
    if ((fl & LB_ALL_OPAQUE) && !(fl & LB_EMISSIVE)) {   // opaque_for_light_computation
        const_cast<uint32_t *>(P.scene.light)[idx] = TX_OPAQUE;
        if (!queue) return;
        mark_changed(P, idx);
        P.pending[idx] = 0;
    } else {
        if (!queue) return;
        P.pending[idx] = PRIO_NEWLY_VISIBLE;
    }
    int x, y, z;
    cube_of(P.scene, idx, x, y, z);
#pragma unroll
    for (int f = 0; f < 6; f++) {
        const int s = (f < 3) ? -1 : 1, a = f % 3, opp = (f < 3) ? f + 3 : f - 3;
        uint32_t nidx;
        if (!cube_index(P.scene, x + (a == 0 ? s : 0), y + (a == 1 ? s : 0), z + (a == 2 ? s : 0), &nidx)) continue;
        if (!((__ldg(&P.blocks[block_id_at(P.scene, nidx)].flags) >> opp) & 1u)) P.pending[nidx] = PRIO_NEWLY_VISIBLE;
    }
}

// modified_cube for a cube that holds block `id`, if `id` is one of the redefined indices (`s_mask`, one bit per block
// index).
__device__ __forceinline__ void relight_cube(const LightParams &P, const uint32_t *s_mask, uint32_t idx, uint32_t id,
                                             uint32_t queue) {
    if ((s_mask[id >> 5] >> (id & 31u)) & 1u) modified_cube(P, idx, id, queue);
}

// The light rule of aicb_light_edit_region, after k_region_cells wrote the box's cells and marked in `mask` the cubes
// whose block changed: modified_cube for each of those, one cube of the box per thread (consecutive threads take
// consecutive cubes of a row, so their cell, flag and pending accesses coalesce).  Mutation::set applies the rule cube by
// cube, each reading the neighbours' blocks of that moment; run against the final cells it leaves the same queue and
// texels.  A changed cube ends OPAQUE and unqueued, or queued at NEWLY_VISIBLE, whatever its neighbours did.  An unchanged
// or not yet edited neighbour shows the rule its final block; a neighbour edited later is queued by its own edit unless
// it becomes opaque for light, and then it is opaque on every face, so the rule on its final block does not queue it.
__global__ void __launch_bounds__(256) k_region_light(const LightParams P, const RegionBox box, const uint32_t *mask,
                                                      uint32_t volume, uint32_t queue) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= volume || !((__ldg(mask + (p >> 5)) >> (p & 31u)) & 1u)) return;
    const uint32_t row = p / box.size[2], rx = row / box.size[1], ry = row - rx * box.size[1];
    const uint32_t idx = ((box.lo[0] + rx) * (uint32_t)P.scene.size[1] + box.lo[1] + ry) * (uint32_t)P.scene.size[2] +
                         box.lo[2] + (p - row * box.size[2]);
    modified_cube(P, idx, block_id_at(P.scene, idx), queue);
}

// One changing entry of an aicb_light_edit_cubes list (its id differs from the block its cube holds at that point of
// the list), as staged: the cube's Z-major index, the entry's id, and the block the cube holds after the whole list.
struct __align__(8) EditEntry {
    uint32_t idx;
    uint16_t id;
    uint16_t final_id;
};
static_assert(sizeof(EditEntry) == 8, "an EditEntry is staged as 8 bytes");

// The cells of a list of sets: every changing entry stores its cube's final cell word, the kind from the block table's
// records on the device.  A cube named by several entries has them all store the same word.
template <bool WIDE>
__global__ void __launch_bounds__(256) k_edit_cells(const DeviceScene S, const EditEntry *entries, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const EditEntry e = entries[i];
    const uint32_t word = e.final_id | (__ldg(&S.blocks[e.final_id].kind_res) & 0xffu) << (WIDE ? 16 : 14);
    if (WIDE) ((uint32_t *)S.cells)[e.idx] = word;
    else ((uint16_t *)S.cells)[e.idx] = (uint16_t)word;
}

// The light rule of aicb_light_edit_cubes, after k_edit_cells wrote the final cells: one changing entry per thread.
// A cube's own queue entry, and its neighbours', are k_region_light's argument: its last changing entry decides them and
// sets its final block, so modified_cube against the final cells is exact.  The texels are not a function of the final
// cells: every changing entry whose own block is opaque for light stores OPAQUE and enters the set, as the reference's
// set does even when a later entry makes the cube non-opaque again (A -> B -> A keeps an OPAQUE texel).  Every write
// stores OPAQUE, 0 or NEWLY_VISIBLE where no other thread stores a different value.
__global__ void __launch_bounds__(256) k_edit_light(const LightParams P, const EditEntry *entries, uint32_t n,
                                                    uint32_t queue) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const EditEntry e = entries[i];
    const uint32_t fl = __ldg(&P.blocks[e.id].flags);
    if ((fl & LB_ALL_OPAQUE) && !(fl & LB_EMISSIVE)) {   // opaque_for_light_computation
        const_cast<uint32_t *>(P.scene.light)[e.idx] = TX_OPAQUE;
        if (queue) mark_changed(P, e.idx);
    }
    modified_cube(P, e.idx, block_id_at(P.scene, e.idx), queue);
}

// The staging of a device edit list (light_edit_cubes_device) over the list sorted stably by cube (stage_cube_list):
// (keys, vals) = (cube, list position) in sorted order, so a cube's entries form a run in list order.  What the host
// loop of light_edit_cubes finds, as three passes and two scans:
//   - k_stage_changing: an entry changes iff its id differs from the one before it in its run, or for a run's first
//     entry from its cube's cell (the host mirror's value then); `head` marks the runs' first entries.
//   - k_stage_final: the last entry of each run (run = the inclusive sum of head) gives its cube's final id.
//   - k_stage_entries: each changing entry at its rank among the changing entries in list order (pos, the exclusive
//     sum of `changing`), as the host loop stages it; v->count is their number.
// A cube out of bounds sorts as cube 0 and is never applied (its call is rejected).
__global__ void __launch_bounds__(256) k_stage_changing(const DeviceScene S, const uint32_t *__restrict__ keys,
                                                        const uint32_t *__restrict__ vals, const uint16_t *__restrict__ ids,
                                                        uint32_t n, uint32_t volume, uint32_t *__restrict__ head,
                                                        uint32_t *__restrict__ changing) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t key = keys[p], i = vals[p];
    const bool first = p == 0 || keys[p - 1] != key;
    const uint32_t before = !first ? (uint32_t)ids[vals[p - 1]] : key < volume ? block_id_at(S, key) : 0u;
    head[p] = first ? 1u : 0u;
    changing[i] = ids[i] != before ? 1u : 0u;
}

__global__ void __launch_bounds__(256) k_stage_final(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                     const uint16_t *__restrict__ ids, const uint32_t *__restrict__ run,
                                                     uint32_t n, uint16_t *__restrict__ run_final) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n || (p + 1 < n && keys[p + 1] == keys[p])) return;
    run_final[run[p] - 1] = ids[vals[p]];
}

__global__ void __launch_bounds__(256) k_stage_entries(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                       const uint16_t *__restrict__ ids, const uint32_t *__restrict__ run,
                                                       const uint16_t *__restrict__ run_final,
                                                       const uint32_t *__restrict__ changing,
                                                       const uint32_t *__restrict__ pos, uint32_t n,
                                                       EditEntry *__restrict__ entries, InputVerdict *v) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    if (p == 0) v->count = pos[n - 1] + changing[n - 1];
    const uint32_t i = vals[p];
    if (changing[i]) entries[pos[i]] = EditEntry{keys[p], ids[i], run_final[run[p] - 1]};
}

// The scan of aicb_light_relight_blocks: every cell of the scene, 16 bytes per load (8 u16 cells or 4 u32 cells,
// decoded as block_id_at does), against the redefined indices in shared memory (65 536 bits).  Grid-stride; the cells
// past the last whole vector are read one by one.
constexpr uint32_t RELIGHT_MASK_WORDS = 65536 / 32;
__global__ void __launch_bounds__(256) k_relight_blocks(const LightParams P, const uint32_t *mask, uint32_t queue) {
    __shared__ uint32_t s_mask[RELIGHT_MASK_WORDS];
    for (uint32_t i = threadIdx.x; i < RELIGHT_MASK_WORDS; i += blockDim.x) s_mask[i] = mask[i];
    __syncthreads();
    const DeviceScene &S = P.scene;
    const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    const uint4 *cells = (const uint4 *)S.cells;
    const uint32_t per = S.wide_cells ? 4u : 8u, n_vec = P.volume / per;
    for (uint32_t v = t0; v < n_vec; v += stride) {
        const uint4 c = __ldg(cells + v);
        const uint32_t w[4] = {c.x, c.y, c.z, c.w}, base = v * per;
        if (S.wide_cells) {
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) relight_cube(P, s_mask, base + k, w[k] & 0xffffu, queue);
        } else {
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                relight_cube(P, s_mask, base + 2 * k, w[k] & 0x3fffu, queue);
                relight_cube(P, s_mask, base + 2 * k + 1, (w[k] >> 16) & 0x3fffu, queue);
            }
        }
    }
    for (uint32_t idx = n_vec * per + t0; idx < P.volume; idx += stride) relight_cube(P, s_mask, idx, block_id_at(S, idx), queue);
}

// A box of cubes as offsets from the scene's lower corner (hi exclusive), already clipped to the bounds.
struct QueueBox {
    uint32_t lo[3], hi[3];
};

// LightUpdateQueue::insert (queue.rs:107-133) at one priority, raise-only, for a set of cubes: those whose texel is
// Uninitialized (UNINIT: the load rule of Space::new_from_builder, space.rs:290-313) or those in `box`
// (light_needs_update_in_region, updater.rs:122-133).  One 256-thread block per queue tile, grid-stride over the tiles
// [tile0, tile1); a thread owns 4 consecutive cubes: one word of pending bytes and, for UNINIT, one 16-byte load of
// their texels.  No other thread writes the word, so no CAS.  A tile with a selected cube has its bound raised to
// `prio`, which k_gather reads; the selected cubes are counted into counters->queued.
template <bool UNINIT>
__global__ void __launch_bounds__(256) k_queue_cubes(const LightParams P, uint32_t tile0, uint32_t tile1, QueueBox box,
                                                     uint32_t prio) {
    __shared__ uint32_t s_n[8];
    const DeviceScene &S = P.scene;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t total = 0;   // (thread 0) the block's selected cubes
    for (uint32_t tile = tile0 + blockIdx.x; tile < tile1; tile += gridDim.x) {
        const uint32_t w = tile * (LIGHT_TILE / 4) + threadIdx.x, base = w * 4;
        uint32_t sel = 0;
        if (base < P.volume) {
            if (UNINIT) {
                uint32_t t[4];
                if (base + 4 <= P.volume) {
                    const uint4 v = __ldg((const uint4 *)S.light + w);
                    t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w;
                } else {
#pragma unroll
                    for (uint32_t k = 0; k < 4; k++) t[k] = base + k < P.volume ? S.light[base + k] : TX_NO_RAYS;
                }
#pragma unroll
                for (uint32_t k = 0; k < 4; k++) sel |= ((t[k] >> 24) == 0 ? 1u : 0u) << k;   // LightStatus::Uninitialized
            } else {
                const uint32_t sy = (uint32_t)S.size[1], sz = (uint32_t)S.size[2];
                uint32_t z = base % sz, y = (base / sz) % sy, x = base / sz / sy;
#pragma unroll
                for (uint32_t k = 0; k < 4; k++) {
                    const bool in = base + k < P.volume && x >= box.lo[0] && x < box.hi[0] && y >= box.lo[1] &&
                                    y < box.hi[1] && z >= box.lo[2] && z < box.hi[2];
                    sel |= (in ? 1u : 0u) << k;
                    if (++z == sz) {
                        z = 0;
                        if (++y == sy) { y = 0; x++; }
                    }
                }
            }
            if (sel) {
                uint32_t *wp = (uint32_t *)P.pending + w;
                const uint32_t old = *wp;
                uint32_t nv = old;
#pragma unroll
                for (uint32_t k = 0; k < 4; k++)
                    if (((sel >> k) & 1u) && ((old >> (8 * k)) & 255u) < prio) nv = (nv & ~(255u << (8 * k))) | (prio << (8 * k));
                if (nv != old) *wp = nv;
            }
        }
        const uint32_t n = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(sel));
        if (lane == 0) s_n[wid] = n;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t c = 0;
            for (int i = 0; i < 8; i++) c += s_n[i];
            if (c && P.tile_max[tile] < prio) P.tile_max[tile] = prio;
            total += c;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0 && total) atomicAdd(&P.counters->queued, total);
}

// Taking the set of changed cubes: an ordered stream compaction of the bitmap.  A chunk is the CHANGES_CHUNK_WORDS
// words of bits (32 768 cubes) one 256-thread block reads, four consecutive words per thread.
constexpr uint32_t CHANGES_CHUNK_WORDS = 1024;

// The exclusive prefix of `v` over the block's 256 threads, in thread order; the block's total in *total.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t s_part[8];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
        if ((int)lane >= off) inc += t;
    }
    if (lane == 31) s_part[wid] = inc;
    __syncthreads();
    uint32_t before = 0, sum = 0;
    for (uint32_t k = 0; k < 8; k++) {
        if (k < wid) before += s_part[k];
        sum += s_part[k];
    }
    *total = sum;
    return before + inc - v;
}

// 1. the number of changed cubes in each chunk
__global__ void __launch_bounds__(256) k_changes_count(const uint32_t *bits, uint32_t n_words, uint32_t *chunk_sums) {
    const uint32_t w0 = blockIdx.x * CHANGES_CHUNK_WORDS + threadIdx.x * 4u;
    uint32_t c = 0;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) c += w0 + k < n_words ? __popc(bits[w0 + k]) : 0u;
    uint32_t total;
    block_exclusive_scan(c, &total);
    if (threadIdx.x == 0) chunk_sums[blockIdx.x] = total;
}

// 2. one block of 1024 threads: the chunk sums become each chunk's first output position, in place, and
// chunk_sums[n_chunks] the size of the set
__global__ void __launch_bounds__(1024) k_changes_scan(uint32_t *chunk_sums, uint32_t n_chunks) {
    __shared__ uint32_t s_part[32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t per = (n_chunks + 1023u) / 1024u, c0 = threadIdx.x * per;
    uint32_t run = 0;
    for (uint32_t c = c0; c < c0 + per && c < n_chunks; c++) run += chunk_sums[c];
    uint32_t inc = run;
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
        if ((int)lane >= off) inc += t;
    }
    if (lane == 31) s_part[wid] = inc;
    __syncthreads();
    uint32_t at = inc - run;
    for (uint32_t k = 0; k < wid; k++) at += s_part[k];
    for (uint32_t c = c0; c < c0 + per && c < n_chunks; c++) {
        const uint32_t v = chunk_sums[c];
        chunk_sums[c] = at;
        at += v;
    }
    if (threadIdx.x == 1023) chunk_sums[n_chunks] = at;
}

// 3. every changed cube's index, in increasing order, and its texel as it is now; the words read are cleared
__global__ void __launch_bounds__(256) k_changes_emit(uint32_t *bits, uint32_t n_words, const uint32_t *chunk_starts,
                                                       const uint32_t *light, uint32_t *out_indices, uint32_t *out_texels) {
    const uint32_t w0 = blockIdx.x * CHANGES_CHUNK_WORDS + threadIdx.x * 4u;
    uint32_t word[4], c = 0;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        word[k] = w0 + k < n_words ? bits[w0 + k] : 0u;
        c += __popc(word[k]);
    }
    uint32_t total;
    uint32_t at = chunk_starts[blockIdx.x] + block_exclusive_scan(c, &total);
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        uint32_t b = word[k];
        if (!b) continue;
        bits[w0 + k] = 0u;
        while (b) {
            const uint32_t idx = (w0 + k) * 32u + (uint32_t)(__ffs(b) - 1);
            b &= b - 1u;
            out_indices[at] = idx;
            out_texels[at] = light[idx];
            at++;
        }
    }
}

// The rounds of a budgeted step (aicb_light_update_from_queue) gather with these kernels in place of k_gather.  A round
// whose band (the cubes k_gather would take) fits in the budget left takes the band.  A round that does not fit takes the
// budget's worth of it: by priority, highest first, and within the priority where the budget ends (the cut level),
// lowest index first.  Which cubes a round takes thus depends on the queue alone, never on the order blocks run in.
// Everything stays on the device, behind the round's k_find_max:
//   1. k_step_band: the band's cubes per priority, over the tiles k_gather would read;
//   2. k_step_cut (one thread): the whole band, or the cut level and how many of its cubes to take; the round's list
//      length, taken from the budget;
//   3. only when a round may cut: k_step_level counts each tile's cubes at the cut level, and k_changes_scan turns the
//      counts into the rank of each tile's first such cube;
//   4. k_step_emit: the taken cubes into the list, their pending bytes cleared, each tile's bound lowered to what stays,
//      as k_gather does.
// A round that starts with no budget left or nothing above epsilon gathers nothing and leaves the bounds alone.
struct LightStepCut {
    uint32_t hist[PRIORITY_BAND + 1];   // the band's cubes at priority `priority - k` (k_step_cut clears it)
    uint32_t active;                    // this round gathers
    uint32_t level;                     // the cut level; 0 when the round takes its whole band
    uint32_t take;                      // cubes of the cut level the round takes
    uint32_t emitted;                   // list entries k_step_emit has placed
};

// the tiles k_gather reads in a round of priority `prio`, and the cubes it takes from them (block-uniform / per cube)
__device__ __forceinline__ bool band_tile(const LightParams &P, uint32_t tile, uint32_t prio) {
    const uint32_t tm = P.tile_max[tile];
    return tm > P.epsilon_priority && tm + PRIORITY_BAND >= prio;
}
__device__ __forceinline__ bool in_band(const LightParams &P, uint32_t p, uint32_t prio) {
    return p > P.epsilon_priority && p <= prio && p + PRIORITY_BAND >= prio;
}

__global__ void __launch_bounds__(256) k_step_band(const LightParams P, uint32_t n_tiles, LightStepCut *cut) {
    __shared__ uint32_t s_hist[PRIORITY_BAND + 1];
    const uint32_t prio = P.counters->priority;
    if (P.counters->budget == 0 || prio <= P.epsilon_priority) return;
    for (uint32_t i = threadIdx.x; i <= PRIORITY_BAND; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const uint32_t n_words = (P.volume + 3) / 4;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (!band_tile(P, tile, prio)) continue;   // (block-uniform)
        const uint32_t w = tile * (LIGHT_TILE / 4) + threadIdx.x;
        const uint32_t v = w < n_words ? ((const uint32_t *)P.pending)[w] : 0u;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            const uint32_t p = (v >> (8 * k)) & 255u;
            const bool in = in_band(P, p, prio) && w * 4 + k < P.volume;
            // one shared atomic per distinct level of the warp
            const uint32_t key = in ? prio - p : 0xffu;
            const uint32_t same = __match_any_sync(0xffffffffu, key);
            if (in && (threadIdx.x & 31) == (uint32_t)(__ffs(same) - 1)) atomicAdd(&s_hist[key], (uint32_t)__popc(same));
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i <= PRIORITY_BAND; i += blockDim.x)
        if (s_hist[i]) atomicAdd(&cut->hist[i], s_hist[i]);
}

__global__ void k_step_cut(const LightParams P, LightStepCut *cut) {
    const uint32_t prio = P.counters->priority;
    unsigned long long left = P.counters->budget;
    const bool active = left != 0 && prio > P.epsilon_priority;
    uint32_t level = 0, take = 0, taken = 0;
    for (uint32_t k = 0; k <= PRIORITY_BAND; k++) {
        const uint32_t h = cut->hist[k];
        cut->hist[k] = 0u;
        if (!active || level) continue;
        if (h > left) {   // the budget ends inside this level
            level = prio - k;
            take = (uint32_t)left;
        } else {
            left -= h;
        }
        taken += level ? take : h;
    }
    cut->active = active ? 1u : 0u;
    cut->level = level;
    cut->take = take;
    cut->emitted = 0u;
    if (!active) return;
    P.counters->gathered = taken;
    P.counters->budget = level ? 0ull : left;
}

__global__ void __launch_bounds__(256) k_step_level(const LightParams P, uint32_t n_tiles, const LightStepCut *cut,
                                                    uint32_t *counts) {
    if (!cut->active || !cut->level) return;
    const uint32_t prio = P.counters->priority, level = cut->level;
    const uint32_t n_words = (P.volume + 3) / 4;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        uint32_t c = 0;
        if (band_tile(P, tile, prio)) {
            const uint32_t w = tile * (LIGHT_TILE / 4) + threadIdx.x;
            const uint32_t v = w < n_words ? ((const uint32_t *)P.pending)[w] : 0u;
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) c += (((v >> (8 * k)) & 255u) == level && w * 4 + k < P.volume) ? 1u : 0u;
        }
        uint32_t total;
        block_exclusive_scan(c, &total);
        if (threadIdx.x == 0) counts[tile] = total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_step_emit(const LightParams P, uint32_t n_tiles, LightStepCut *cut,
                                                   const uint32_t *level_starts) {
    __shared__ uint8_t s_sel[LIGHT_TILE / 4];
    __shared__ uint32_t s_max[8], s_base;
    if (!cut->active) return;
    const uint32_t prio = P.counters->priority, level = cut->level, take = cut->take;
    const uint32_t n_words = (P.volume + 3) / 4;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t wl = list_word_of_thread(P);
    uint32_t *pending = (uint32_t *)P.pending;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (!band_tile(P, tile, prio)) continue;   // (block-uniform)
        // which cubes of the tile the round takes: one word per thread in index order, for the rank in the cut level
        {
            const uint32_t w = tile * (LIGHT_TILE / 4) + threadIdx.x;
            const uint32_t v = w < n_words ? pending[w] : 0u;
            uint32_t sel = 0, at_level = 0;
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                const uint32_t p = (v >> (8 * k)) & 255u;
                if (!in_band(P, p, prio) || w * 4 + k >= P.volume) continue;
                if (p > level) sel |= 1u << k;
                else if (p == level) at_level |= 1u << k;
            }
            if (level) {   // (block-uniform)
                uint32_t total;
                uint32_t rank = level_starts[tile] + block_exclusive_scan((uint32_t)__popc(at_level), &total);
#pragma unroll
                for (uint32_t k = 0; k < 4; k++)
                    if (at_level & (1u << k)) {
                        if (rank < take) sel |= 1u << k;
                        rank++;
                    }
            }
            s_sel[threadIdx.x] = (uint8_t)sel;
        }
        __syncthreads();
        // the list, in k_gather's thread layout
        const uint32_t w = tile * (LIGHT_TILE / 4) + wl;
        uint32_t v = w < n_words ? pending[w] : 0u;
        const uint32_t sel = s_sel[wl], cnt = (uint32_t)__popc(sel);
        uint32_t total;
        const uint32_t before = block_exclusive_scan(cnt, &total);
        uint32_t rest = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) if (!(sel & (1u << k))) rest = max(rest, (v >> (8 * k)) & 255u);
        rest = __reduce_max_sync(0xffffffffu, rest);
        if (lane == 0) s_max[wid] = rest;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t m = 0;
            for (int i = 0; i < 8; i++) m = max(m, s_max[i]);
            s_base = total ? atomicAdd(&cut->emitted, total) : 0u;
            P.tile_max[tile] = m;
        }
        __syncthreads();
        if (cnt) {
            uint32_t at = s_base + before;
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)
                if (sel & (1u << k)) { P.list[at++] = w * 4 + k; v &= ~(255u << (8 * k)); }
            pending[w] = v;
        }
        __syncthreads();
    }
}

// The queue as a budgeted step leaves it: the queued cubes and their highest priority, exact (the tile bounds are upper
// bounds only), from the pending bytes, 16 per load.
__global__ void __launch_bounds__(256) k_queue_summary(const LightParams P) {
    uint32_t n = 0, m = 0;
    const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    const uint32_t n_vec = P.volume / 16;
    for (uint32_t i = t0; i < n_vec; i += stride) {
        const uint4 q = ((const uint4 *)P.pending)[i];
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            n += (uint32_t)__popc(__vcmpne4(w[k], 0u)) / 8u;   // (0xff per byte that differs)
            const uint32_t h = __vmaxu4(w[k], w[k] >> 16);
            m = max(m, max(h & 255u, (h >> 8) & 255u));
        }
    }
    for (uint32_t idx = n_vec * 16 + t0; idx < P.volume; idx += stride) {
        const uint32_t p = P.pending[idx];
        n += p ? 1u : 0u;
        m = max(m, p);
    }
    n = __reduce_add_sync(0xffffffffu, n);
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) {
        if (n) atomicAdd(&P.counters->queue_len, n);
        if (m) atomicMax(&P.counters->queue_max, m);
    }
}

// Packing the rays of aicb_light_compute_debug.  A cube's rays are the records of the walk that computed its texel:
// the chain walk's, or the lockstep walk's where the chain walk overflowed.
__device__ __forceinline__ bool ray_counts_for_its_cube(const LightRayRecord &r, const uint8_t *lockstep) {
    return ((r.item & LIGHT_RAY_LOCKSTEP) != 0) == (lockstep[r.item & ~LIGHT_RAY_LOCKSTEP] != 0);
}

// 1. each cube's number of rays (k_changes_scan then turns the counts into each cube's first output position)
__global__ void __launch_bounds__(256) k_rays_count(const LightRayRecord *recs, uint32_t n_recs, const uint8_t *lockstep,
                                                    uint32_t *counts) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_recs; j += gridDim.x * blockDim.x)
        if (ray_counts_for_its_cube(recs[j], lockstep)) atomicAdd(counts + (recs[j].item & ~LIGHT_RAY_LOCKSTEP), 1u);
}

// 2. every counted record into its cube's range, in any order
__global__ void __launch_bounds__(256) k_rays_place(const LightRayRecord *recs, uint32_t n_recs, const uint8_t *lockstep,
                                                    const uint32_t *starts, uint32_t *fill, LightRayRecord *placed) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_recs; j += gridDim.x * blockDim.x) {
        const LightRayRecord r = recs[j];
        if (!ray_counts_for_its_cube(r, lockstep)) continue;
        const uint32_t c = r.item & ~LIGHT_RAY_LOCKSTEP;
        placed[starts[c] + atomicAdd(fill + c, 1u)] = r;
    }
}

// 3. one warp per cube: each ray goes to its rank by chart node within the cube's range (nodes are distinct per cube)
__global__ void __launch_bounds__(256) k_rays_order(const LightRayRecord *placed, const uint32_t *starts, uint32_t n_cubes,
                                                    aicb_light_ray *out) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n_cubes; c += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t s = starts[c], m = starts[c + 1] - s;
        for (uint32_t j = lane; j < m; j += 32) {
            const uint32_t node = placed[s + j].node;
            uint32_t rank = 0;
            for (uint32_t k = 0; k < m; k++) rank += placed[s + k].node < node ? 1u : 0u;
            out[s + rank] = placed[s + j].ray;
        }
    }
}

// Replica i's parameters: its own field, blocks, chart, term slots and overflow list with its count; replica 0's queue,
// round buffers, counters and sets (peer pointers on the other replicas).  Replica 0 takes both parts from itself.
LightParams light_params(Replicas r, size_t i) {
    const aicb_scene *s = r.scene[i];
    const LightState::Own &own = s->light.own;
    const LightState::Shared &root = r.scene[0]->light.shared;
    const LightChart &chart = r.ctx[i]->light_chart;
    LightParams P;
    std::memset(&P, 0, sizeof P);
    P.scene = s->ds;
    P.blocks = s->blocks.light.get<LightBlockDev>();
    P.chart_pre = chart.pre.get<LightNodePre>();
    P.sky_term = own.sky_term.get<float4>();
    P.chains = chart.chains.get<LightChain>();
    P.node_rel = chart.node_rel.get<uchar4>();
    P.euler = chart.euler.get<uint16_t>();
    P.n_chains = chart.n_chains;
    P.n_euler = chart.n_euler;
    P.term_scratch = chart.term_scratch.get<float4>();
    P.overflow = own.overflow.get<uint32_t>();
    P.chart_nodes = chart.nodes;
    P.tile_max = root.tile_max.get<uint32_t>();
    P.changed = r.scene[0]->light.changed();
    P.pending = root.pending.get<uint8_t>();
    P.list = root.list.get<uint32_t>();
    P.new_light = root.new_light.get<uint32_t>();
    P.diff = root.diff.get<uint8_t>();
    P.counters = root.counters.get<LightCounters>();
    P.overflow_count = i == 0 ? &P.counters->overflow : own.overflow_count.get<uint32_t>();
    P.dirty = root.dirty.get<uint32_t>();
    P.changes = root.changes.get<uint32_t>();
    P.volume = (uint32_t)s->host->volume;
    P.max_distance = s->host->light_max_distance;
    return P;
}

// end_of_ray (updater.rs:889-924) without the lane's alpha and bundle weight: per chart node, the sky light its bundle
// collects from a BlockSky with these faces (texels NX..PZ) — the same f32 operations, in the same order, as the
// reference evaluates per ray end.  LightState::Own::sky_term.
std::vector<float4> sky_terms(const uint32_t sky_faces[6]) {
    const std::vector<LightNodePre> &pre = chart_preorder_host();
    float lut[256];
    lut[0] = 0.0f;
    for (int i = 1; i < 256; i++) lut[i] = (float)std::exp2((double)(((float)i - 144.0f) / 10.0f));
    auto psc = [](float v) { return v > 0.0f ? v : 0.0f; };
    auto psm = [](float a, float b) { float v = a * b; return (v != v) ? 0.0f : v; };
    std::vector<float4> sky(pre.size());
    for (size_t k = 0; k < pre.size(); k++) {
        const float *cw = pre[k].w;
        float t[6][3];
        for (int f = 0; f < 6; f++) {
            const uint32_t tx = sky_faces[f];
            const float kk = psc(cw[f]);
            t[f][0] = psm(lut[tx & 255], kk);
            t[f][1] = psm(lut[(tx >> 8) & 255], kk);
            t[f][2] = psm(lut[(tx >> 16) & 255], kk);
        }
        const float kr = psc(1.0f / ((cw[0] + cw[3]) + (cw[1] + cw[4]) + (cw[2] + cw[5])));
        float c[3];
        for (int i = 0; i < 3; i++) c[i] = psm((t[0][i] + t[3][i]) + (t[1][i] + t[4][i]) + (t[2][i] + t[5][i]), kr);
        sky[k] = make_float4(c[0], c[1], c[2], 0.0f);
    }
    return sky;
}

// Every replica's light state and, on a group, replica 0's push targets: the other replicas' light volumes.  A replica
// that has no own part yet takes `terms` as its sky_term, or the scene's sky tabulated once for every such replica.
aicb_status ensure_replicas(Replicas r, const std::vector<float4> *terms = nullptr) {
    std::vector<float4> tabulated;
    for (size_t i = 0; i < r.n; i++) {
        if (!terms && !r.scene[i]->light.own.sky_term) {
            tabulated = sky_terms(r.scene[0]->ds.sky_faces);
            terms = &tabulated;
        }
        CU(cudaSetDevice(r.ctx[i]->device));
        TRY(r.scene[i]->light.ensure(r.scene[i], i, r.n, terms));
    }
    if (r.n == 1) return AICB_OK;
    std::vector<uint32_t *> targets;
    for (size_t i = 1; i < r.n; i++) targets.push_back(const_cast<uint32_t *>(r.scene[i]->ds.light));
    CU(cudaSetDevice(r.ctx[0]->device));
    CU(cudaMemcpy(r.scene[0]->light.shared.push_targets.get(), targets.data(), targets.size() * sizeof(uint32_t *),
                  cudaMemcpyHostToDevice));
    // device 0 writes the other replicas' volumes: after what their streams hold (aicb_scene_update_cubes is queued)
    return fan_in(r.ctx, r.n);
}

// Every replica's walk of one form, replica i against its own field on its own context: the compute form (the round's
// list, or the n `explicit_cubes`) with the lockstep walk of the overflow it met, or the mark form.  On a group the
// walks start behind device 0's stream, and device 0's stream waits for them.
aicb_status walk(Replicas r, const std::vector<LightParams> &RP, bool mark, uint32_t n = 0,
                 const int32_t *explicit_cubes = nullptr) {
    const bool group = r.n > 1;
    if (group) TRY(fan_out(r.ctx, r.n));
    for (size_t i = 0; i < r.n; i++) {
        aicb_ctx *c = r.ctx[i];
        cudaStream_t cs = c->stream.get();
        if (group) CU(cudaSetDevice(c->device));
        if (mark) {
            k_walk_chains<true><<<c->light_chart.walk_blocks, 128, 0, cs>>>(RP[i], 0, nullptr);
            continue;
        }
        if (i > 0) CU(cudaMemsetAsync(RP[i].overflow_count, 0, 4, cs));   // (replica 0's: with its other counters)
        k_walk_chains<false><<<c->light_chart.walk_blocks, 128, 0, cs>>>(RP[i], n, explicit_cubes);
        k_compute_overflow<<<c->num_sms * 8, 128, 0, cs>>>(RP[i], explicit_cubes);
    }
    return group ? fan_in(r.ctx, r.n) : AICB_OK;
}

// A round restarts the counters of its list (gathered, priority) and of its walks (changed .. overflow).
constexpr size_t ROUND_LIST_COUNTERS = offsetof(LightCounters, max_diff);
constexpr size_t ROUND_WALK_COUNTERS =
    offsetof(LightCounters, overflow) + sizeof(uint32_t) - offsetof(LightCounters, changed);

// evaluate_light (space.rs:1496-1527): rounds until the highest queued priority is <= from_difference(epsilon).
// A round: device 0 gathers the cubes of the round's band from its queue; every replica walks a share of them against
// its own field (compute form + the overflow it met), taking cubes from device 0's counter and writing device 0's
// results; device 0 applies them; on a group it pushes the segments it wrote to the other replicas; every replica
// then walks a share of the changed cubes (mark form), raising priorities in device 0's queue.  Compute is Jacobi
// within a round and marks merge by max, so a group performs one context's operations.  One context issues no event
// and no push.
// `budget` (a budgeted step, light_update_from_queue): every queued priority is eligible, the rounds gather with the
// k_step_* kernels, and they stop once *budget cube updates are made or the queue is empty.  The budget left lives in
// the device counters, so a batch's rounds stay queued back to back; a round after it runs out gathers nothing.
// nullptr: evaluate_light(epsilon)'s rounds.
aicb_status propagate(Replicas r, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff, uint64_t *node_visits,
                      const uint64_t *budget = nullptr) {
    aicb_scene *s = r.scene[0];
    aicb_ctx *ctx = s->ctx;
    cudaStream_t st = ctx->stream.get();
    const bool group = r.n > 1;
    std::vector<LightParams> RP;
    for (size_t i = 0; i < r.n; i++) {
        RP.push_back(light_params(r, i));
        RP.back().epsilon_priority = budget ? 0u : (uint32_t)epsilon / 2 + 1;
    }
    const LightParams &P = RP[0];
    const int blocks = ctx->num_sms * 8;
    const int wide = ctx->num_sms * 8;    // 128-thread blocks of k_compute_overflow and k_apply (grid-stride)
    const uint32_t n_tiles = (uint32_t)((s->host->volume + LIGHT_TILE - 1) / LIGHT_TILE);
    LightStepCut *cut = s->light.shared.step.get<LightStepCut>();
    uint32_t *level_starts = (uint32_t *)(cut + 1);
    uint64_t total = 0, visits = 0, rounds = 0;
    uint32_t maxd = 0;
    CU(cudaEventRecord(ctx->ev_light[0].get(), st));
    CU(cudaMemsetAsync(P.counters, 0, sizeof(LightCounters), st));
    if (budget) {
        CU(cudaMemcpyAsync(&P.counters->budget, budget, sizeof *budget, cudaMemcpyHostToDevice, st));
        CU(cudaMemsetAsync(cut, 0, sizeof(LightStepCut), st));
    }
    k_tile_rebuild<<<blocks, 256, 0, st>>>(P, n_tiles);   // (fast_evaluate / edits write the priority bytes directly)
    const int ROUNDS_PER_SYNC = 8;
    uint64_t left = budget ? *budget : 1;   // (the budget left at the last synchronisation)
    for (int batch = 0; batch < 100000 && left; batch++) {
        // a round takes at most the volume, so with this much left no round of the batch can cut
        const bool may_cut = left < (uint64_t)ROUNDS_PER_SYNC * s->host->volume;
        for (int round = 0; round < ROUNDS_PER_SYNC; round++) {
            CU(cudaMemsetAsync(P.counters, 0, ROUND_LIST_COUNTERS, st));
            CU(cudaMemsetAsync(&P.counters->changed, 0, ROUND_WALK_COUNTERS, st));
            k_find_max<<<16, 256, 0, st>>>(P, n_tiles);
            if (!budget) {
                k_gather<<<blocks, 256, 0, st>>>(P, n_tiles);
            } else {
                k_step_band<<<blocks, 256, 0, st>>>(P, n_tiles, cut);
                k_step_cut<<<1, 1, 0, st>>>(P, cut);
                if (may_cut) {
                    k_step_level<<<blocks, 256, 0, st>>>(P, n_tiles, cut, level_starts);
                    k_changes_scan<<<1, 1024, 0, st>>>(level_starts, n_tiles);
                }
                k_step_emit<<<blocks, 256, 0, st>>>(P, n_tiles, cut, level_starts);
            }
            TRY(walk(r, RP, false));
            if (group) k_apply<true><<<wide, 128, 0, st>>>(P);
            else k_apply<false><<<wide, 128, 0, st>>>(P);
            k_compact_changed<<<blocks, 256, 0, st>>>(P);
            if (group)
                k_push<<<blocks, 256, 0, st>>>(P, s->light.shared.push_targets.get<uint32_t *const>(),
                                               (uint32_t)(r.n - 1));
            TRY(walk(r, RP, true));   // (on a group, the next round's queue holds every replica's marks)
        }
        LightCounters h;
        CU(cudaMemcpyAsync(&h, P.counters, sizeof h, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        CU(cudaGetLastError());
        total = h.updates;
        visits = h.node_visits;
        maxd = h.max_diff;
        rounds += ROUNDS_PER_SYNC;
        if (budget) left = h.budget;
        if (h.priority <= P.epsilon_priority) break;   // the batch's last round found nothing above epsilon
    }
    CU(cudaEventRecord(ctx->ev_light[1].get(), st));
    CU(cudaEventSynchronize(ctx->ev_light[1].get()));
    float ms = 0.0f;
    CU(cudaEventElapsedTime(&ms, ctx->ev_light[0].get(), ctx->ev_light[1].get()));
    s->host->light_stats[0] = total;
    s->host->light_stats[1] = visits;
    s->host->light_stats[2] = rounds;
    s->host->light_stats[3] = (uint64_t)(ms * 1000.0f);   // device time of the propagation in microseconds
    if (updates_done) *updates_done = total;
    if (max_diff) *max_diff = (uint8_t)maxd;
    if (node_visits) *node_visits = visits;
    return AICB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// a scene's light state (internal.h)
// ---------------------------------------------------------------------------------------------
// What aicb_scene_device_bytes counts of a light state's parts (it leaves out the tile bounds, the step's cut, the
// counters, the overflow count and the push targets).
static size_t change_bytes(size_t vol) { return (vol + 31) / 32 * 4; }
static size_t dirty_bytes(size_t vol) { return (vol + 1023) / 1024 * 4 + 16; }
static uint64_t own_bytes(size_t vol) { return chart_preorder_host().size() * sizeof(float4) + vol * 4; }
static uint64_t shared_bytes(size_t vol, bool group) { return vol * 10 + change_bytes(vol) + (group ? dirty_bytes(vol) : 0); }

aicb_status LightState::ensure(aicb_scene *s, size_t replica, size_t n_replicas, const std::vector<float4> *terms) {
    if (s->host->light_max_distance == 0) return aicb_fail(AICB_ERR_INVALID, "scene has LightPhysics::None (light_max_distance == 0)");
    TRY(ensure_chart(s->ctx));
    const size_t vol = s->host->volume;
    const bool add_own = !own.sky_term, add_shared = replica == 0 && !shared.pending, group = n_replicas > 1;
    DeviceBuffer light;
    Own o;
    Shared sh;
    if (!s->d_light) {  // a scene created without a light volume starts all NO_RAYS (initialize_light, updater.rs:628-656)
        const std::vector<uint32_t> init(vol, TX_NO_RAYS);
        TRY(light.upload(init.data(), vol * 4, 16));
    }
    if (add_own) {
        TRY(o.sky_term.upload(terms ? *terms : sky_terms(s->ds.sky_faces)));
        TRY(o.overflow.ensure(vol * 4 + 16));
        if (replica > 0) TRY(o.overflow_count.ensure(4));
    }
    if (add_shared) {
        TRY(sh.pending.ensure(vol + 16));
        CU(cudaMemset(sh.pending.get(), 0, vol + 16));
        TRY(sh.tile_max.ensure(((vol + LIGHT_TILE - 1) / LIGHT_TILE + 1) * 4));
        TRY(sh.step.ensure(sizeof(LightStepCut) + ((vol + LIGHT_TILE - 1) / LIGHT_TILE + 1) * 4));
        TRY(sh.list.ensure(vol * 4 + 16));
        TRY(sh.new_light.ensure(vol * 4 + 16));
        TRY(sh.diff.ensure(vol + 16));
        TRY(sh.counters.ensure(sizeof(LightCounters)));
        TRY(sh.changes.ensure(change_bytes(vol)));
        CU(cudaMemset(sh.changes.get(), 0, change_bytes(vol)));
        if (group) {
            TRY(sh.dirty.ensure(dirty_bytes(vol)));
            CU(cudaMemset(sh.dirty.get(), 0, dirty_bytes(vol)));
            TRY(sh.push_targets.ensure((n_replicas - 1) * sizeof(uint32_t *)));
        }
    }
    if (light) {
        s->d_light = std::move(light);
        s->ds.light = s->d_light.get<uint32_t>();
        s->device_bytes += vol * 4;
    }
    if (add_own) {
        own = std::move(o);
        s->device_bytes += own_bytes(vol);
    }
    if (add_shared) {
        shared = std::move(sh);
        s->device_bytes += shared_bytes(vol, group);
    }
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// the light calls over a scene's replicas (internal.h): one context's entry points below, a group's in group.cu
// ---------------------------------------------------------------------------------------------
aicb_status light_fast_evaluate(Replicas r) {
    TRY(ensure_replicas(r));
    aicb_scene *s = r.scene[0];
    cudaStream_t stream = s->ctx->stream.get();
    LightParams P = light_params(r, 0);
    const uint32_t cols = (uint32_t)s->ds.size[0] * (uint32_t)s->ds.size[2];
    if (cols) k_fast_evaluate<<<(cols + 127) / 128, 128, 0, stream>>>(P);
    CU(cudaGetLastError());
    // the other replicas take the whole volume once (peer copies)
    for (size_t i = 1; i < r.n; i++)
        CU(cudaMemcpyAsync(r.scene[i]->d_light.get(), s->d_light.get(), s->host->volume * 4, cudaMemcpyDefault, stream));
    CU(cudaStreamSynchronize(stream));
    return AICB_OK;
}

// The cubes are split across the replicas by device 0's work counter; every replica computes the overflow of its own
// walks; the outputs are device 0's, in input order.
aicb_status light_compute(Replicas r, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]) {
    aicb_scene *s = r.scene[0];
    if (n && (!cubes || !out)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > s->host->volume) return aicb_fail(AICB_ERR_INVALID, "more cubes than the Space holds");
    TRY(ensure_replicas(r));
    if (!n) return AICB_OK;
    std::vector<LightParams> RP;
    for (size_t i = 0; i < r.n; i++) RP.push_back(light_params(r, i));
    const LightParams &P = RP[0];
    cudaStream_t stream = s->ctx->stream.get();
    DeviceBuffer d_cubes;   // on device 0; the other replicas read it over peer access
    TRY(d_cubes.upload(cubes, n * 12));
    CU(cudaMemsetAsync(P.counters, 0, sizeof(LightCounters), stream));
    TRY(walk(r, RP, false, (uint32_t)n, d_cubes.get<int32_t>()));
    LightCounters h;
    CU(cudaMemcpyAsync(out, P.new_light, n * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(&h, P.counters, sizeof h, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    uint64_t overflowed = h.overflow;
    for (size_t i = 1; i < r.n; i++) {   // (every replica's stream is done: device 0's waited for them)
        uint32_t c = 0;
        CU(cudaMemcpy(&c, RP[i].overflow_count, 4, cudaMemcpyDeviceToHost));
        overflowed += c;
    }
    s->host->light_stats[0] = n;
    s->host->light_stats[1] = h.node_visits;
    s->host->light_stats[2] = overflowed;   // cubes that took the lockstep walk (a chain with more terms than its slots)
    s->host->light_stats[3] = 0;
    return AICB_OK;
}

// Replica 0 walks every cube with the recording walks, then the rays are counted, scanned, placed and put in chart
// order on the device.  The log starts with room for 256 rays a cube; a call that finds more runs the walks again with
// room for all of them (the walks are deterministic).  Nothing is copied to the caller before the capacity check.
aicb_status light_compute_debug(Replicas r, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4], aicb_light_ray *rays,
                                size_t capacity, uint32_t *ray_counts, size_t *n_rays_total) {
    aicb_scene *s = r.scene[0];
    if (!n_rays_total || (n && (!cubes || !out || !ray_counts))) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > s->host->volume) return aicb_fail(AICB_ERR_INVALID, "more cubes than the Space holds");
    for (size_t i = 0; i < n; i++)
        for (int a = 0; a < 3; a++)
            if ((uint32_t)(cubes[i][a] - s->ds.lo[a]) >= (uint32_t)s->ds.size[a])
                return aicb_fail(AICB_ERR_INVALID, "cube out of the Space's bounds");
    TRY(ensure_replicas(r));
    if (!rays) capacity = 0;
    if (!n) {
        *n_rays_total = 0;
        return AICB_OK;
    }
    const Replicas r0{r.scene, r.ctx, 1};
    const LightParams P = light_params(r0, 0);
    aicb_ctx *ctx = s->ctx;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream.get();
    DeviceBuffer d_cubes, d_lockstep, d_count, d_recs;
    TRY(d_cubes.upload(cubes, n * 12));
    TRY(d_lockstep.ensure(n));
    TRY(d_count.ensure(4));
    uint32_t n_recs = (uint32_t)std::min<size_t>(n * 256, (size_t)1 << 22);
    LightCounters h;
    for (;;) {
        TRY(d_recs.ensure((size_t)n_recs * sizeof(LightRayRecord)));
        const LightRayLog log{d_recs.get<LightRayRecord>(), d_count.get<uint32_t>(), d_lockstep.get<uint8_t>(), n_recs};
        CU(cudaMemsetAsync(P.counters, 0, sizeof(LightCounters), st));
        CU(cudaMemsetAsync(log.count, 0, 4, st));
        k_walk_chains_record<<<ctx->light_chart.walk_blocks, 128, 0, st>>>(P, (uint32_t)n, d_cubes.get<int32_t>(), log);
        k_compute_overflow_record<<<ctx->num_sms * 8, 128, 0, st>>>(P, d_cubes.get<int32_t>(), log);
        CU(cudaGetLastError());
        uint32_t logged = 0;
        CU(cudaMemcpyAsync(&logged, log.count, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(&h, P.counters, sizeof h, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (logged <= n_recs) {
            n_recs = logged;
            break;
        }
        n_recs = logged;
    }
    // k_changes_scan scans any array of counts: starts[c] = the first ray of cube c, starts[n] = the total
    DeviceBuffer d_starts, d_fill;
    TRY(d_starts.ensure((n + 1) * 4));
    TRY(d_fill.ensure(n * 4));
    CU(cudaMemsetAsync(d_starts.get(), 0, (n + 1) * 4, st));
    const int wide = ctx->num_sms * 8;
    const uint8_t *lockstep = d_lockstep.get<uint8_t>();
    if (n_recs) k_rays_count<<<wide, 256, 0, st>>>(d_recs.get<LightRayRecord>(), n_recs, lockstep, d_starts.get<uint32_t>());
    k_changes_scan<<<1, 1024, 0, st>>>(d_starts.get<uint32_t>(), (uint32_t)n);
    CU(cudaGetLastError());
    std::vector<uint32_t> starts(n + 1);
    std::vector<uint32_t> texels(n);
    CU(cudaMemcpyAsync(starts.data(), d_starts.get(), (n + 1) * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(texels.data(), P.new_light, n * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const size_t total = starts[n];
    *n_rays_total = total;
    if (capacity < total)
        return aicb_fail(AICB_ERR_INVALID, "ray_capacity is smaller than the number of rays (*n_rays_total)");
    if (total) {
        DeviceBuffer d_placed, d_rays;
        TRY(d_placed.ensure(total * sizeof(LightRayRecord)));
        TRY(d_rays.ensure(total * sizeof(aicb_light_ray)));
        CU(cudaMemsetAsync(d_fill.get(), 0, n * 4, st));
        k_rays_place<<<wide, 256, 0, st>>>(d_recs.get<LightRayRecord>(), n_recs, lockstep, d_starts.get<uint32_t>(),
                                           d_fill.get<uint32_t>(), d_placed.get<LightRayRecord>());
        k_rays_order<<<wide, 256, 0, st>>>(d_placed.get<LightRayRecord>(), d_starts.get<uint32_t>(), (uint32_t)n,
                                           d_rays.get<aicb_light_ray>());
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(rays, d_rays.get(), total * sizeof(aicb_light_ray), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    std::memcpy(out, texels.data(), n * 4);
    for (size_t i = 0; i < n; i++) ray_counts[i] = starts[i + 1] - starts[i];
    // aicb_light_compute's counters: the walks' are the same on one context or a group
    s->host->light_stats[0] = n;
    s->host->light_stats[1] = h.node_visits;
    s->host->light_stats[2] = h.overflow;
    s->host->light_stats[3] = 0;
    return AICB_OK;
}

aicb_status light_evaluate(Replicas r, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                           uint64_t *node_visits) {
    TRY(ensure_replicas(r));
    return propagate(r, epsilon, updates_done, max_diff, node_visits);
}

// update_light_from_queue (updater.rs:180-290) with a count budget: propagate's budgeted rounds, then the queue as they
// left it, counted on the device (k_queue_summary).  A zero budget runs no round.
aicb_status light_update_from_queue(Replicas r, uint64_t max_updates, aicb_light_updates_info *info) {
    TRY(ensure_replicas(r));
    uint64_t updates = 0;
    uint8_t maxd = 0;
    TRY(propagate(r, 0, &updates, &maxd, nullptr, &max_updates));
    aicb_scene *s = r.scene[0];
    cudaStream_t st = s->ctx->stream.get();
    const LightParams P = light_params(r, 0);
    CU(cudaMemsetAsync(&P.counters->queue_len, 0, 2 * sizeof(uint32_t), st));
    k_queue_summary<<<s->ctx->num_sms * 4, 256, 0, st>>>(P);
    CU(cudaGetLastError());
    uint32_t q[2] = {0, 0};
    CU(cudaMemcpyAsync(q, &P.counters->queue_len, sizeof q, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (info) {
        std::memset(info, 0, sizeof *info);
        info->update_count = updates;
        info->queue_count = q[0];
        info->max_update_difference = maxd;
        info->max_queue_priority = (uint8_t)q[1];
    }
    return AICB_OK;
}

// Mutation::set x n (space.rs:1346-1352 -> side_effects_of_set -> modified_cube_needs_update, updater.rs:135-173)
// without propagation.  The list is validated and indexed before anything changes.  One pass in list order over the
// host mirror finds the changing entries (the same-block skip) and writes the mirror, which
// aicb_scene_update_blocks re-encodes cells from; a second pass gives each its cube's final block.  They are staged,
// 8 bytes each, in every replica's context, behind the cube updates queued there: k_edit_cells writes the final cells
// and k_edit_light applies the rule (DESIGN.md §4b).  Replica 0 alone touches the queue and the set.
aicb_status light_edit_cubes(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                             size_t *n_changed) {
    if (n && (!cubes || !new_ids)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > 0xffffffffull) return aicb_fail(AICB_ERR_INVALID, "more than 2^32 - 1 edits");
    SpaceHost &h = *r.scene[0]->host;
    const DeviceScene &ds = r.scene[0]->ds;
    std::vector<uint32_t> idx(n);
    for (size_t i = 0; i < n; i++) {
        const uint32_t dx = (uint32_t)(cubes[i][0] - ds.lo[0]), dy = (uint32_t)(cubes[i][1] - ds.lo[1]),
                       dz = (uint32_t)(cubes[i][2] - ds.lo[2]);
        if (dx >= (uint32_t)ds.size[0] || dy >= (uint32_t)ds.size[1] || dz >= (uint32_t)ds.size[2])
            return aicb_fail(AICB_ERR_INVALID, "cube out of bounds");
        if (new_ids[i] >= h.block_count()) return aicb_fail(AICB_ERR_INVALID, "block id out of range");
        idx[i] = (dx * (uint32_t)ds.size[1] + dy) * (uint32_t)ds.size[2] + dz;
    }
    TRY(ensure_replicas(r));
    if (n_changed) *n_changed = 0;
    if (n == 0) return AICB_OK;
    const size_t room = n * sizeof(EditEntry);
    for (size_t k = 0; k < r.n; k++) {   // every replica's staging is free before any mirror changes
        CU(cudaSetDevice(r.ctx[k]->device));
        TRY(delta_room(r.ctx[k], room));
    }
    TRY(refresh_mirror(r.scene[0]));
    EditEntry *staged = r.ctx[0]->h_delta.get<EditEntry>();
    uint32_t m = 0;
    for (size_t i = 0; i < n; i++) {
        if (h.h_ids[idx[i]] == new_ids[i]) continue;   // Mutation::set of the same block changes nothing
        h.h_ids[idx[i]] = new_ids[i];
        staged[m++] = EditEntry{idx[i], new_ids[i], 0};
    }
    for (uint32_t k = 0; k < m; k++) staged[k].final_id = h.h_ids[staged[k].idx];
    const size_t bytes = (size_t)m * sizeof(EditEntry);
    for (size_t k = 0; m && k < r.n; k++) {
        aicb_scene *sk = r.scene[k];
        aicb_ctx *c = r.ctx[k];
        cudaStream_t stream = c->stream.get();
        CU(cudaSetDevice(c->device));
        if (k > 0) std::memcpy(c->h_delta.get(), staged, bytes);
        const EditEntry *d_entries = c->d_delta.get<const EditEntry>();
        CU(cudaMemcpyAsync(c->d_delta.get(), c->h_delta.get(), bytes, cudaMemcpyHostToDevice, stream));
        const unsigned blocks = (m + 255) / 256;
        if (sk->ds.wide_cells) k_edit_cells<true><<<blocks, 256, 0, stream>>>(sk->ds, d_entries, m);
        else k_edit_cells<false><<<blocks, 256, 0, stream>>>(sk->ds, d_entries, m);
        k_edit_light<<<blocks, 256, 0, stream>>>(light_params(r, k), d_entries, m, k == 0);
        CU(cudaGetLastError());
        CU(cudaEventRecord(c->ev_delta.get(), stream));   // renders on other streams wait for it (launch_trace)
    }
    for (size_t k = 0; m && k < r.n; k++) {
        CU(cudaSetDevice(r.ctx[k]->device));
        CU(cudaStreamSynchronize(r.ctx[k]->stream.get()));
    }
    CU(cudaSetDevice(r.ctx[0]->device));
    if (n_changed) *n_changed = m;
    return AICB_OK;
}

// light_edit_cubes with the list in device memory: checked and staged on replica 0's device (stage_cube_list, then
// k_stage_*), so that the EditEntry list is the host loop's; only the verdict and its length come back.  Every replica
// then applies it as light_edit_cubes does, the others from a peer copy of replica 0's list.  The host mirror is left
// stale.
aicb_status light_edit_cubes_device(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                                    size_t *n_changed, cudaStream_t caller) {
    if (n && (!cubes || !new_ids)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > 0xffffffffull) return aicb_fail(AICB_ERR_INVALID, "more than 2^32 - 1 edits");
    aicb_scene *s0 = r.scene[0];
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    uint32_t m = 0;
    const EditEntry *d_entries = nullptr;
    if (n) {
        TRY(check_device_pointer(cubes, c0->device, false, 4, "cubes"));
        TRY(check_device_pointer(new_ids, c0->device, false, 2, "new_ids"));
        TRY(join_caller(r.ctx, 1, caller));
        const uint32_t nn = (uint32_t)n;
        cudaStream_t stream = c0->stream.get();
        size_t scan_in = 0, scan_ex = 0;
        CU(cub::DeviceScan::InclusiveSum(nullptr, scan_in, (uint32_t *)nullptr, (uint32_t *)nullptr, nn, stream));
        CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_ex, (uint32_t *)nullptr, (uint32_t *)nullptr, nn, stream));
        const size_t a = ((size_t)nn * 4 + 255) & ~(size_t)255, b = ((size_t)nn * 2 + 255) & ~(size_t)255;
        CubeList l;
        TRY(stage_cube_list(s0, cubes, new_ids, nn, 4 * a + b + (size_t)nn * sizeof(EditEntry),
                            std::max(scan_in, scan_ex), &l));
        char *x = (char *)l.extra;
        uint32_t *head = (uint32_t *)x, *run = (uint32_t *)(x + a), *changing = (uint32_t *)(x + 2 * a),
                 *pos = (uint32_t *)(x + 3 * a);
        uint16_t *run_final = (uint16_t *)(x + 4 * a);
        EditEntry *entries = (EditEntry *)(x + 4 * a + b);
        const unsigned blocks = (nn + 255) / 256;
        k_stage_changing<<<blocks, 256, 0, stream>>>(s0->ds, l.keys, l.vals, new_ids, nn, (uint32_t)s0->host->volume,
                                                     head, changing);
        size_t tb = l.temp_bytes;
        CU(cub::DeviceScan::InclusiveSum(l.temp, tb, head, run, nn, stream));
        k_stage_final<<<blocks, 256, 0, stream>>>(l.keys, l.vals, new_ids, run, nn, run_final);
        tb = l.temp_bytes;
        CU(cub::DeviceScan::ExclusiveSum(l.temp, tb, changing, pos, nn, stream));
        k_stage_entries<<<blocks, 256, 0, stream>>>(l.keys, l.vals, new_ids, run, run_final, changing, pos, nn, entries,
                                                    l.verdict);
        CU(cudaGetLastError());
        TRY(read_verdict(c0, l.verdict, &m));
        d_entries = entries;
    }
    TRY(ensure_replicas(r));
    if (n_changed) *n_changed = 0;
    if (n == 0) return AICB_OK;
    for (size_t k = 0; m && k < r.n; k++) {
        aicb_scene *sk = r.scene[k];
        aicb_ctx *c = r.ctx[k];
        cudaStream_t stream = c->stream.get();
        CU(cudaSetDevice(c->device));
        void *from = const_cast<EditEntry *>(d_entries);
        if (k > 0) TRY(copy_to_replica(r, k, d_entries, (size_t)m * sizeof(EditEntry), &from));
        const EditEntry *e = (const EditEntry *)from;
        const unsigned blocks = (m + 255) / 256;
        if (sk->ds.wide_cells) k_edit_cells<true><<<blocks, 256, 0, stream>>>(sk->ds, e, m);
        else k_edit_cells<false><<<blocks, 256, 0, stream>>>(sk->ds, e, m);
        k_edit_light<<<blocks, 256, 0, stream>>>(light_params(r, k), e, m, k == 0);
        CU(cudaGetLastError());
        CU(cudaEventRecord(c->ev_delta.get(), stream));   // renders on other streams wait for it (launch_trace)
    }
    for (size_t k = 0; m && k < r.n; k++) {
        CU(cudaSetDevice(r.ctx[k]->device));
        CU(cudaStreamSynchronize(r.ctx[k]->stream.get()));
    }
    if (m) s0->host->ids_stale = true;
    CU(cudaSetDevice(c0->device));
    if (n_changed) *n_changed = m;
    return release_caller(c0, caller);
}

// light_edit_cubes, then evaluate_light(epsilon).
aicb_status light_edit_and_propagate(Replicas r, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n_edits,
                                     uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff) {
    TRY(light_edit_cubes(r, cubes, new_ids, n_edits, nullptr));
    return propagate(r, epsilon, updates_done, max_diff, nullptr);
}

// modified_cube_needs_update (updater.rs:135-173) for every cube that holds one of the indices, with the block's current
// definition, then evaluate_light(epsilon).  The cubes are found on the device (k_relight_blocks), on every replica
// against its own cells, ordered on each replica's stream behind the cube updates queued there; only replica 0 holds
// the queue and the set of changed cubes.
aicb_status light_relight_blocks(Replicas r, const uint16_t *indices, size_t n, uint8_t epsilon,
                                 uint64_t *updates_done, uint8_t *max_diff) {
    if (n && !indices) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    aicb_scene *s = r.scene[0];
    std::vector<uint32_t> mask(RELIGHT_MASK_WORDS, 0u);
    for (size_t i = 0; i < n; i++) {
        if (indices[i] >= s->host->block_count()) return aicb_fail(AICB_ERR_INVALID, "block index out of range");
        mask[indices[i] >> 5] |= 1u << (indices[i] & 31u);
    }
    TRY(ensure_replicas(r));
    if (n) {
        std::vector<DeviceBuffer> d_mask(r.n);
        for (size_t i = 0; i < r.n; i++) {
            aicb_ctx *c = r.ctx[i];
            cudaStream_t stream = c->stream.get();
            CU(cudaSetDevice(c->device));
            TRY(d_mask[i].ensure(mask.size() * 4));
            CU(cudaMemcpyAsync(d_mask[i].get(), mask.data(), mask.size() * 4, cudaMemcpyHostToDevice, stream));
            k_relight_blocks<<<c->num_sms * 8, 256, 0, stream>>>(light_params(r, i), d_mask[i].get<uint32_t>(), i == 0);
            CU(cudaGetLastError());
        }
        for (size_t i = 0; i < r.n; i++) {
            CU(cudaSetDevice(r.ctx[i]->device));
            CU(cudaStreamSynchronize(r.ctx[i]->stream.get()));
        }
        CU(cudaSetDevice(s->ctx->device));
    }
    return propagate(r, epsilon, updates_done, max_diff, nullptr);
}

// Mutation::fill / fill_uniform(region) (space.rs:1392-1412, 1455-1479): Mutation::set for every cube of the box.  On
// every replica, behind the cube updates queued on its stream: the cells (region_cells), the changed cubes marked in
// the replica's overflow list (a round buffer, empty between light calls: one bit per cube of the box), then the light
// rule on the device (k_region_light).  Replica 0 alone counts the changed cubes and touches the queue and the set; the
// host mirror takes the ids once.  Nothing propagates; the tile bounds are rebuilt from the pending bytes by the next
// propagation.  This is the body of the host and the device form, after validation: the ids are a host array (staged,
// and the host mirror takes them) or, with on_device, device memory every replica reads where it is (the mirror is then
// marked stale).
static aicb_status edit_region(Replicas r, const RegionBox &box, const uint16_t *ids, uint16_t uniform_id, bool on_device,
                               size_t *n_changed) {
    TRY(ensure_replicas(r));
    if (n_changed) *n_changed = 0;
    const size_t vol = box.volume();
    if (vol == 0) return AICB_OK;
    if (!on_device) TRY(refresh_mirror(r.scene[0]));
    uint32_t edited = 0;
    for (size_t i = 0; i < r.n; i++) {
        aicb_ctx *c = r.ctx[i];
        cudaStream_t stream = c->stream.get();
        CU(cudaSetDevice(c->device));
        const LightParams P = light_params(r, i);
        if (i == 0) CU(cudaMemsetAsync(&P.counters->edited, 0, 4, stream));
        TRY(region_cells(r.scene[i], box, ids, uniform_id, nullptr, on_device, P.overflow,
                         i == 0 ? &P.counters->edited : nullptr));
        k_region_light<<<(unsigned)((vol + 255) / 256), 256, 0, stream>>>(P, box, P.overflow, (uint32_t)vol, i == 0);
        CU(cudaGetLastError());
        CU(cudaEventRecord(c->ev_delta.get(), stream));   // renders on other streams wait for it (launch_trace)
        if (i == 0) CU(cudaMemcpyAsync(&edited, &P.counters->edited, 4, cudaMemcpyDeviceToHost, stream));
    }
    if (on_device) r.scene[0]->host->ids_stale = true;
    else mirror_region(*r.scene[0]->host, r.scene[0]->ds, box, ids, uniform_id);
    for (size_t i = 0; i < r.n; i++) {
        CU(cudaSetDevice(r.ctx[i]->device));
        CU(cudaStreamSynchronize(r.ctx[i]->stream.get()));
    }
    CU(cudaSetDevice(r.ctx[0]->device));
    if (n_changed) *n_changed = edited;
    return AICB_OK;
}

aicb_status light_edit_region(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                              size_t *n_changed) {
    RegionBox box;
    TRY(check_region(r.scene[0], region, ids, uniform_id, &box));
    return edit_region(r, box, ids, uniform_id, false, n_changed);
}

aicb_status light_edit_region_device(Replicas r, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                     size_t *n_changed, cudaStream_t caller) {
    RegionBox box;
    TRY(check_region_device(r, region, ids, uniform_id, nullptr, caller, &box));
    TRY(edit_region(r, box, ids, uniform_id, ids != nullptr, n_changed));
    return release_caller(r.ctx[0], caller);
}

// LightStorage::maybe_reinitialize_for_physics_change (space/light/updater.rs:80-113):
//   - the sky: every replica takes it, and a replica's sky_term is re-tabulated (once per call) where the BlockSky's
//     faces changed.  Nothing else changes for the sky alone (the reference's "TODO: if only sky color is different").
//   - Rays of another distance: every replica's state, allocated where it has none (LightState::ensure), then
//     fast_evaluate_light with the new sky on device 0, copied to the others.  It writes every texel and every queue
//     entry, so initialize_light's uniform fill is never observable and is not made.  Every cube enters the set of
//     changed cubes: the whole volume was replaced.
//   - None: every replica's light volume and state are freed (frames read PackedLight::ONE; the set goes with them).
// The allocation comes first and is the only step that can fail for want of memory: a failure frees what it allocated
// and leaves every replica as it was.
aicb_status light_set_physics(Replicas r, const DeviceScene &sky, uint32_t max_distance) {
    aicb_scene *s0 = r.scene[0];
    SpaceHost &h = *s0->host;
    const bool relight = max_distance != h.light_max_distance;
    const bool new_faces = std::memcmp(sky.sky_faces, s0->ds.sky_faces, sizeof sky.sky_faces) != 0;
    std::vector<float4> terms;
    if (new_faces || (relight && max_distance)) terms = sky_terms(sky.sky_faces);
    if (relight && max_distance) {
        struct Before {
            bool light, own, shared;
            uint64_t device_bytes;
        };
        std::vector<Before> before;
        for (size_t i = 0; i < r.n; i++) {
            aicb_scene *s = r.scene[i];
            before.push_back({(bool)s->d_light, (bool)s->light.own.sky_term, (bool)s->light.shared.pending,
                              s->device_bytes});
        }
        const uint32_t before_max = h.light_max_distance;
        h.light_max_distance = max_distance;
        const aicb_status st = ensure_replicas(r, &terms);
        if (st != AICB_OK) {
            for (size_t i = 0; i < r.n; i++) {
                aicb_scene *s = r.scene[i];
                cudaSetDevice(r.ctx[i]->device);
                if (!before[i].light) {
                    s->d_light.reset();
                    s->ds.light = nullptr;
                }
                if (!before[i].own) s->light.own = LightState::Own();
                if (!before[i].shared) s->light.shared = LightState::Shared();
                s->device_bytes = before[i].device_bytes;
            }
            h.light_max_distance = before_max;
            cudaSetDevice(s0->ctx->device);
            return st;
        }
    }
    for (size_t i = 0; i < r.n; i++) {
        aicb_scene *s = r.scene[i];
        DeviceScene &ds = s->ds;
        CU(cudaSetDevice(r.ctx[i]->device));
        std::memcpy(ds.sky_faces, sky.sky_faces, sizeof ds.sky_faces);
        ds.sky_mean = sky.sky_mean;
        ds.sky_kind = sky.sky_kind;
        std::memcpy(ds.sky_colors, sky.sky_colors, sizeof ds.sky_colors);
        if (new_faces && s->light.own.sky_term)
            CU(cudaMemcpy(s->light.own.sky_term.get(), terms.data(), terms.size() * sizeof(float4), cudaMemcpyHostToDevice));
        if (relight && !max_distance) {
            const size_t vol = h.volume;
            if (s->d_light) s->device_bytes -= vol * 4;
            if (s->light.own.sky_term) s->device_bytes -= own_bytes(vol);
            if (s->light.shared.pending) s->device_bytes -= shared_bytes(vol, (bool)s->light.shared.dirty);
            s->light.own = LightState::Own();
            s->light.shared = LightState::Shared();
            s->d_light.reset();
            ds.light = nullptr;
        }
    }
    h.light_max_distance = max_distance;
    CU(cudaSetDevice(s0->ctx->device));
    if (!relight || !max_distance) return AICB_OK;
    TRY(light_fast_evaluate(r));
    // every cube is changed: whole words of the bitmap, then the cubes of a last, partial word
    uint32_t *changes = s0->light.shared.changes.get<uint32_t>();
    cudaStream_t stream = s0->ctx->stream.get();
    const size_t whole = h.volume / 32;
    const uint32_t tail = (1u << (h.volume % 32)) - 1u;
    CU(cudaMemsetAsync(changes, 0xff, whole * 4, stream));
    if (tail) CU(cudaMemcpyAsync(changes + whole, &tail, 4, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));
    return AICB_OK;
}

// k_queue_cubes on replica 0 (its texels, its queue), behind the work queued on its context: the cube updates and
// uploads whose texels the load rule reads.  *n_queued: the cubes selected.
static aicb_status queue_cubes(Replicas r, bool uninit, const QueueBox &box, uint8_t priority, size_t *n_queued) {
    aicb_scene *s = r.scene[0];
    const LightParams P = light_params(r, 0);
    cudaStream_t st = s->ctx->stream.get();
    uint32_t tile0 = 0, tile1 = (uint32_t)((s->host->volume + LIGHT_TILE - 1) / LIGHT_TILE);
    if (!uninit) {   // the tiles from the box's first cube to its last
        const uint32_t sy = (uint32_t)s->ds.size[1], sz = (uint32_t)s->ds.size[2];
        tile0 = ((box.lo[0] * sy + box.lo[1]) * sz + box.lo[2]) / LIGHT_TILE;
        tile1 = (((box.hi[0] - 1) * sy + box.hi[1] - 1) * sz + box.hi[2] - 1) / LIGHT_TILE + 1;
    }
    const uint32_t blocks = std::min(tile1 - tile0, (uint32_t)s->ctx->num_sms * 32u);
    CU(cudaMemsetAsync(&P.counters->queued, 0, 4, st));
    if (uninit) k_queue_cubes<true><<<blocks, 256, 0, st>>>(P, tile0, tile1, box, priority);
    else k_queue_cubes<false><<<blocks, 256, 0, st>>>(P, tile0, tile1, box, priority);
    CU(cudaGetLastError());
    uint32_t n = 0;
    CU(cudaMemcpyAsync(&n, &P.counters->queued, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n_queued) *n_queued = n;
    return AICB_OK;
}

// Space::new_from_builder's load rule (space.rs:290-313): every cube of replica 0's volume whose texel is
// Uninitialized enters the queue at Priority::UNINIT.  No texel is written and nothing propagates.
aicb_status light_queue_uninitialized(Replicas r, size_t *n_queued) {
    TRY(ensure_replicas(r));
    return queue_cubes(r, true, QueueBox{}, PRIO_UNINIT, n_queued);
}

// LightStorage::light_needs_update_in_region (updater.rs:122-133): every cube of region ∩ bounds at `priority`.  Its
// sweep branch (more than 400 cubes) queues the same cubes at the same priority.
aicb_status light_queue_region(Replicas r, const aicb_aab *region, uint8_t priority) {
    if (!region) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (priority == 0) return aicb_fail(AICB_ERR_INVALID, "priority 0 (Priority::MIN) never enters the queue");
    TRY(ensure_replicas(r));
    const DeviceScene &ds = r.scene[0]->ds;
    QueueBox box;
    for (int a = 0; a < 3; a++) {
        const int64_t lo = std::max<int64_t>(region->lower[a], ds.lo[a]);
        const int64_t hi = std::min<int64_t>((int64_t)region->lower[a] + region->size[a], (int64_t)ds.lo[a] + ds.size[a]);
        if (hi <= lo) return AICB_OK;   // an empty intersection
        box.lo[a] = (uint32_t)(lo - ds.lo[a]);
        box.hi[a] = (uint32_t)(hi - ds.lo[a]);
    }
    return queue_cubes(r, false, box, priority, nullptr);
}

// The pending bytes are the whole queue between light calls; a scene with no light call yet has an empty queue.
aicb_status light_download_queue(aicb_scene *s, uint8_t *priorities, size_t n_texels, size_t *n_queued) {
    if (!priorities) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n_texels != s->host->volume) return aicb_fail(AICB_ERR_INVALID, "light volume size mismatch");
    if (s->host->light_max_distance == 0) return aicb_fail(AICB_ERR_INVALID, "scene has LightPhysics::None (light_max_distance == 0)");
    if (s->light.shared.pending) {
        CU(cudaSetDevice(s->ctx->device));
        cudaStream_t st = s->ctx->stream.get();
        CU(cudaMemcpyAsync(priorities, s->light.shared.pending.get(), s->host->volume, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    } else {
        std::memset(priorities, 0, s->host->volume);
    }
    if (n_queued) {
        size_t n = 0;
        for (size_t i = 0; i < s->host->volume; i++) n += priorities[i] != 0;
        *n_queued = n;
    }
    return AICB_OK;
}

aicb_status light_download(aicb_scene *s, uint8_t (*out)[4], size_t n_texels) {
    if (!s || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n_texels != s->host->volume) return aicb_fail(AICB_ERR_INVALID, "light volume size mismatch");
    if (!s->d_light) return aicb_fail(AICB_ERR_INVALID, "scene has no light volume (LightPhysics::None)");
    CU(cudaSetDevice(s->ctx->device));
    // ordered behind everything queued on the context's stream (cube deltas, propagation)
    CU(cudaMemcpyAsync(out, s->d_light.get(), s->host->volume * 4, cudaMemcpyDeviceToHost, s->ctx->stream.get()));
    CU(cudaStreamSynchronize(s->ctx->stream.get()));
    return AICB_OK;
}

// aicb_light_download into device memory of replica 0's device: one device-to-device copy on replica 0's stream,
// behind the caller's work and everything queued on the context.
aicb_status light_download_device(Replicas r, uint8_t (*out)[4], size_t n_texels, cudaStream_t caller) {
    aicb_scene *s = r.scene[0];
    if (!out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n_texels != s->host->volume) return aicb_fail(AICB_ERR_INVALID, "light volume size mismatch");
    if (!s->d_light) return aicb_fail(AICB_ERR_INVALID, "scene has no light volume (LightPhysics::None)");
    CU(cudaSetDevice(s->ctx->device));
    if (n_texels == 0) return AICB_OK;
    TRY(check_device_pointer(out, s->ctx->device, false, 4, "out"));
    TRY(join_caller(r.ctx, 1, caller));
    cudaStream_t st = s->ctx->stream.get();
    CU(cudaMemcpyAsync(out, s->d_light.get(), n_texels * 4, cudaMemcpyDeviceToDevice, st));
    if (r.n > 1) CU(cudaStreamSynchronize(st));   // a group call returns with its output final
    return release_caller(s->ctx, caller);
}

// The size of the set of changed cubes (kernels 1 and 2 of the take), behind everything queued on the context's stream;
// the chunks' output positions stay in chunk_sums() for k_changes_emit.
static aicb_status count_changes(const aicb_scene *s, uint32_t *n) {
    const uint32_t n_words = (uint32_t)((s->host->volume + 31) / 32);
    const uint32_t n_chunks = (n_words + CHANGES_CHUNK_WORDS - 1) / CHANGES_CHUNK_WORDS;
    cudaStream_t st = s->ctx->stream.get();
    uint32_t *chunk_sums = s->light.chunk_sums();   // (n_chunks + 1) * 4 <= volume / 8192 + 8 of diff's volume + 16
    k_changes_count<<<n_chunks, 256, 0, st>>>(s->light.shared.changes.get<uint32_t>(), n_words, chunk_sums);
    k_changes_scan<<<1, 1024, 0, st>>>(chunk_sums, n_chunks);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(n, chunk_sums + n_chunks, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return AICB_OK;
}

aicb_status light_changes_count(const aicb_scene *s, size_t *n_changed) {
    if (!n_changed) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (s->host->light_max_distance == 0) return aicb_fail(AICB_ERR_INVALID, "scene has LightPhysics::None (light_max_distance == 0)");
    *n_changed = 0;
    if (!s->light.shared.changes) return AICB_OK;   // no light call yet
    CU(cudaSetDevice(s->ctx->device));
    uint32_t n = 0;
    TRY(count_changes(s, &n));
    *n_changed = n;
    return AICB_OK;
}

// Both outputs: the set, in increasing index order, and the texels as they are now, then the set is empty.  Neither:
// the set is emptied without a copy.  The copy to the caller is queued behind everything on the context's stream.
aicb_status light_take_changes(aicb_scene *s, uint32_t *indices, uint8_t (*texels)[4], size_t capacity, size_t *n_taken) {
    if (!n_taken) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (!indices != !texels) return aicb_fail(AICB_ERR_INVALID, "give both outputs, or neither to discard the set");
    if (s->host->light_max_distance == 0) return aicb_fail(AICB_ERR_INVALID, "scene has LightPhysics::None (light_max_distance == 0)");
    *n_taken = 0;
    if (!s->light.shared.changes) return AICB_OK;
    CU(cudaSetDevice(s->ctx->device));
    cudaStream_t st = s->ctx->stream.get();
    uint32_t n = 0;
    TRY(count_changes(s, &n));
    if (indices && capacity < n) {
        *n_taken = n;
        return aicb_fail(AICB_ERR_INVALID, "capacity is smaller than the set of changed cubes (aicb_light_changes_count)");
    }
    if (n) {
        const uint32_t n_words = (uint32_t)((s->host->volume + 31) / 32);
        if (indices) {
            const uint32_t n_chunks = (n_words + CHANGES_CHUNK_WORDS - 1) / CHANGES_CHUNK_WORDS;
            const LightState &L = s->light;
            k_changes_emit<<<n_chunks, 256, 0, st>>>(L.shared.changes.get<uint32_t>(), n_words, L.chunk_sums(),
                                                      s->ds.light, L.taken_indices(), L.taken_texels());
            CU(cudaMemcpyAsync(indices, L.taken_indices(), (size_t)n * 4, cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(texels, L.taken_texels(), (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        } else {
            CU(cudaMemsetAsync(s->light.shared.changes.get(), 0, (size_t)n_words * 4, st));
        }
        CU(cudaStreamSynchronize(st));
        CU(cudaGetLastError());
    }
    *n_taken = n;
    return AICB_OK;
}

aicb_status light_stats(const aicb_scene *s, uint64_t out[4]) {
    if (!out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    for (int i = 0; i < 4; i++) out[i] = s->host->light_stats[i];
    return AICB_OK;
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

uint32_t aicb_light_chart_chains(uint32_t *preorder, uint32_t (*chains)[6], uint16_t *euler) {
    const ChainTables &t = chain_tables_host();
    if (preorder) {
        std::vector<uint32_t> order;
        build_chart_preorder(build_chart(), &order);
        std::memcpy(preorder, order.data(), order.size() * sizeof(uint32_t));
    }
    if (chains)
        for (size_t c = 0; c < t.chains.size(); c++) {
            const LightChain &ch = t.chains[c];
            chains[c][0] = ch.first_node; chains[c][1] = ch.length; chains[c][2] = ch.n_children;
            chains[c][3] = ch.first_child; chains[c][4] = ch.parent_branch; chains[c][5] = ch.branch;
        }
    if (euler) std::memcpy(euler, t.euler.data(), t.euler.size() * sizeof(uint16_t));
    return (uint32_t)t.chains.size();
}

uint32_t aicb_light_chart(float *weights, uint32_t *children) {
    static const std::vector<LightChartNode> chart = build_chart();
    for (size_t i = 0; i < chart.size(); i++) {
        if (weights) std::memcpy(weights + 6 * i, chart[i].w, 24);
        if (children) std::memcpy(children + 6 * i, chart[i].child, 24);
    }
    return (uint32_t)chart.size();
}

aicb_status aicb_light_fast_evaluate(aicb_scene *s) {
    return on_scene(s, [&](Replicas r) { return light_fast_evaluate(r); });
}

aicb_status aicb_light_compute(aicb_scene *s, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]) {
    return on_scene(s, [&](Replicas r) { return light_compute(r, cubes, n, out); });
}

aicb_status aicb_light_compute_debug(aicb_scene *s, const int32_t (*cubes)[3], size_t n, uint8_t (*out_texels)[4],
                                     aicb_light_ray *rays, size_t ray_capacity, uint32_t *ray_counts,
                                     size_t *n_rays_total) {
    return on_scene(s, [&](Replicas r) {
        return light_compute_debug(r, cubes, n, out_texels, rays, ray_capacity, ray_counts, n_rays_total);
    });
}

aicb_status aicb_light_evaluate(aicb_scene *s, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                                uint64_t *node_visits) {
    return on_scene(s, [&](Replicas r) { return light_evaluate(r, epsilon, updates_done, max_diff, node_visits); });
}

aicb_status aicb_light_update_from_queue(aicb_scene *s, uint64_t max_updates, aicb_light_updates_info *info) {
    return on_scene(s, [&](Replicas r) { return light_update_from_queue(r, max_updates, info); });
}

aicb_status aicb_light_edit_and_propagate(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n_edits,
                                          uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff) {
    return on_scene(s, [&](Replicas r) {
        return light_edit_and_propagate(r, cubes, new_ids, n_edits, epsilon, updates_done, max_diff);
    });
}

aicb_status aicb_light_edit_cubes(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                                  size_t *n_changed) {
    return on_scene(s, [&](Replicas r) { return light_edit_cubes(r, cubes, new_ids, n, n_changed); });
}

aicb_status aicb_light_relight_blocks(aicb_scene *s, const uint16_t *indices, size_t n, uint8_t epsilon,
                                      uint64_t *updates_done, uint8_t *max_diff) {
    return on_scene(s, [&](Replicas r) {
        return light_relight_blocks(r, indices, n, epsilon, updates_done, max_diff);
    });
}

aicb_status aicb_light_edit_region(aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                   size_t *n_changed) {
    return on_scene(s, [&](Replicas r) { return light_edit_region(r, region, ids, uniform_id, n_changed); });
}

aicb_status aicb_light_queue_uninitialized(aicb_scene *s, size_t *n_queued) {
    return on_scene(s, [&](Replicas r) { return light_queue_uninitialized(r, n_queued); });
}

aicb_status aicb_light_queue_region(aicb_scene *s, const aicb_aab *region, uint8_t priority) {
    return on_scene(s, [&](Replicas r) { return light_queue_region(r, region, priority); });
}

aicb_status aicb_light_download_queue(aicb_scene *s, uint8_t *priorities, size_t n_texels, size_t *n_queued) {
    return on_scene(s, [&](Replicas r) { return light_download_queue(r.scene[0], priorities, n_texels, n_queued); });
}

aicb_status aicb_light_download(aicb_scene *s, uint8_t (*out)[4], size_t n_texels) {
    return on_scene(s, [&](Replicas r) { return light_download(r.scene[0], out, n_texels); });
}

aicb_status aicb_light_edit_cubes_device(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                                         size_t *n_changed, void *stream) {
    return on_scene(s, [&](Replicas r) {
        return light_edit_cubes_device(r, cubes, new_ids, n, n_changed, (cudaStream_t)stream);
    });
}

aicb_status aicb_light_edit_region_device(aicb_scene *s, const aicb_aab *region, const uint16_t *ids, uint16_t uniform_id,
                                          size_t *n_changed, void *stream) {
    return on_scene(s, [&](Replicas r) {
        return light_edit_region_device(r, region, ids, uniform_id, n_changed, (cudaStream_t)stream);
    });
}

aicb_status aicb_light_download_device(aicb_scene *s, uint8_t (*out)[4], size_t n_texels, void *stream) {
    return on_scene(s, [&](Replicas r) { return light_download_device(r, out, n_texels, (cudaStream_t)stream); });
}

aicb_status aicb_light_changes_count(const aicb_scene *s, size_t *n_changed) {
    if (!s) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    return light_changes_count(s, n_changed);
}

aicb_status aicb_light_take_changes(aicb_scene *s, uint32_t *indices, uint8_t (*texels)[4], size_t capacity,
                                    size_t *n_taken) {
    return on_scene(s, [&](Replicas r) { return light_take_changes(r.scene[0], indices, texels, capacity, n_taken); });
}

aicb_status aicb_light_stats(const aicb_scene *s, uint64_t out[4]) {
    if (!s) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    return light_stats(s, out);
}
}
