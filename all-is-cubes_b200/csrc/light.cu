// light.cu — host side of the secondary path (SURVEY §8(a) L1-L4): the static light-ray chart
// (space/light/chart/generator.rs), the per-block derived table, and the batched relaxation driver
// replacing LightStorage::update_light_from_queue / apply_light_update / fast_evaluate_light /
// modified_cube_needs_update (space/light/updater.rs) and Mutation::evaluate_light (space.rs:1496-1527).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unordered_map>

#include "internal.h"
#include "light_kernel.cuh"

using namespace aicb;
using namespace aicb_light;

// ---------------------------------------------------------------------------------------------
// chart generation (generator.rs:49-215) — host, once per context
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int CHAIN_WALK_BLOCKS_PER_SM = 6;   // 4 warps, 80 registers, 26 KB of shared memory each

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

void free_chart(aicb_ctx *c) {
    void **ptrs[] = {(void **)&c->d_chart, (void **)&c->d_chart_pre, (void **)&c->d_chains, (void **)&c->d_node_rel,
                     (void **)&c->d_euler, (void **)&c->d_term_scratch};
    for (void **p : ptrs) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
}

aicb_status upload_chart(aicb_ctx *ctx) {
    {
        const ChainTables &t = chain_tables_host();
        if (t.chains.size() > (size_t)LIGHT_MAX_CHAINS || t.chains.size() >= 0x8000u)
            return aicb_fail(AICB_ERR_INVALID, "light chart has more chains than the walk's shared arrays hold");
        size_t branches = 0;
        for (const LightChain &c : t.chains) branches += c.n_children ? 1 : 0;
        if (branches > (size_t)LIGHT_MAX_BRANCHES) return aicb_fail(AICB_ERR_INVALID, "light chart has more branching chains than expected");
        CU(cudaMalloc(&ctx->d_chains, t.chains.size() * sizeof(LightChain)));
        CU(cudaMemcpy(ctx->d_chains, t.chains.data(), t.chains.size() * sizeof(LightChain), cudaMemcpyHostToDevice));
        CU(cudaMalloc(&ctx->d_node_rel, t.node_rel.size() * sizeof(uchar4)));
        CU(cudaMemcpy(ctx->d_node_rel, t.node_rel.data(), t.node_rel.size() * sizeof(uchar4), cudaMemcpyHostToDevice));
        CU(cudaMalloc(&ctx->d_euler, t.euler.size() * sizeof(uint16_t)));
        CU(cudaMemcpy(ctx->d_euler, t.euler.data(), t.euler.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
        ctx->n_chains = (uint32_t)t.chains.size();
        ctx->n_euler = (uint32_t)t.euler.size();
        // one set of term slots per resident warp of the chain walk
        int per_sm = CHAIN_WALK_BLOCKS_PER_SM;
        if (const char *e = getenv("AICB_LIGHT_CTAS")) {   // experiments: fewer resident blocks
            const int v = atoi(e);
            if (v >= 1 && v < per_sm) per_sm = v;
        }
        ctx->chain_walk_blocks = (uint32_t)ctx->num_sms * (uint32_t)per_sm;
        CU(cudaMalloc(&ctx->d_term_scratch, (size_t)ctx->num_sms * CHAIN_WALK_BLOCKS_PER_SM * 4 * LIGHT_WARP_SCRATCH_F4 * sizeof(float4)));
    }
    std::vector<LightChartNode> chart = build_chart();
    const std::vector<LightNodePre> &pre = chart_preorder_host();
    CU(cudaMalloc(&ctx->d_chart_pre, pre.size() * sizeof(LightNodePre)));
    CU(cudaMemcpy(ctx->d_chart_pre, pre.data(), pre.size() * sizeof(LightNodePre), cudaMemcpyHostToDevice));
    CU(cudaMalloc(&ctx->d_chart, chart.size() * sizeof(LightChartNode)));
    CU(cudaMemcpy(ctx->d_chart, chart.data(), chart.size() * sizeof(LightChartNode), cudaMemcpyHostToDevice));
    ctx->chart_nodes = (uint32_t)chart.size();
    return AICB_OK;
}

aicb_status ensure_chart(aicb_ctx *ctx) {
    if (ctx->d_chart) return AICB_OK;   // (d_chart is the last allocation of upload_chart)
    const aicb_status st = upload_chart(ctx);
    if (st != AICB_OK) free_chart(ctx);   // a later call starts over instead of leaking the tables that did fit
    return st;
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
    if ((threadIdx.x & 31) == 0 && m) atomicMax(P.scalars + 1, m);
}

// scalars: [0] cubes gathered this round, [1] highest queued priority this round, [2] largest difference applied
// (accumulated), [3] cube updates (accumulated), [4..5] chart nodes visited (64-bit, accumulated).
// A round's kernels read the round's priority and count from device memory, so rounds are queued back to back
// without a host round trip; a round whose priority is already <= epsilon does nothing.
// One block per tile: the cubes of a tile reach the list in index order (block-wide scan), so 32 consecutive list
// entries are neighbours along z — what the lockstep walk wants.
__global__ void __launch_bounds__(256) k_gather(const LightParams P, uint32_t n_tiles) {
    __shared__ uint32_t s_part[8], s_max[8], s_base;
    const uint32_t prio = P.scalars[1];
    if (prio <= P.epsilon_priority) return;
    const uint32_t n_words = (P.volume + 3) / 4;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // Thread -> word of the tile.  With a power-of-two z extent the tile is a few whole z-rows, and the threads are
    // laid out so that 8 consecutive threads (32 cubes: one warp of the lockstep walk) cover a 4 x 8 patch of (y, z)
    // instead of 32 cubes in a line: neighbours in two directions share more of their chart walk.
    uint32_t wl = threadIdx.x;
    {
        const uint32_t nz = (uint32_t)P.scene.size[2];
        if (nz >= 8 && nz <= 256 && (nz & (nz - 1)) == 0) {
            const uint32_t wpr = nz / 4, q = threadIdx.x >> 3, within = threadIdx.x & 7;
            const uint32_t row_group = q / (wpr / 2), pz = q % (wpr / 2);
            wl = (row_group * 4 + (within >> 1)) * wpr + pz * 2 + (within & 1);
        }
    }
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t tm = P.tile_max[tile];
        if (tm <= P.epsilon_priority || tm + P.priority_band < prio) continue;   // (block-uniform)
        const uint32_t w = tile * (LIGHT_TILE / 4) + wl;
        uint32_t v = w < n_words ? ((uint32_t *)P.pending)[w] : 0u;
        uint32_t sel = 0, cnt = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            const uint32_t p = (v >> (8 * k)) & 255u;
            if (p > P.epsilon_priority && p + P.priority_band >= prio && w * 4 + k < P.volume) { sel |= 1u << k; cnt++; }
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
            s_base = total ? atomicAdd(P.scalars + 0, total) : 0u;
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

// 8 CTAs of 4 warps per SM (64 registers; the records requested ahead spill to L1-resident local memory): the walk is
// latency bound, so 32 resident warps serve it better than the 20 that 94 registers would allow.
#ifndef AICB_LIGHT_MIN_BLOCKS
#define AICB_LIGHT_MIN_BLOCKS 8
#endif
// How many consecutive list entries (neighbouring cubes) one warp walks for together.  The walk is a chain of dependent
// loads per node; a lone warp takes as long per node whatever the number of its lanes that take part.  32 cubes
// share the most node records, but a round of a few ten thousand cubes then occupies a fraction of the resident
// warps and lasts as long as its slowest warp (a 32-cube union of ~20 K nodes).  Narrower batches make more,
// shorter walks: the width is the largest power of two that still yields `P.batches_per_warp` batches per resident warp.
__device__ __forceinline__ uint32_t batch_width(const LightParams &P, uint32_t n, uint32_t n_warps) {
    if (P.batch_width) return P.batch_width;
    uint32_t w = 32;
    while (w > P.min_batch_width && (uint64_t)n < (uint64_t)n_warps * P.batches_per_warp * w) w >>= 1;
    return w;
}

__global__ void __launch_bounds__(128, AICB_LIGHT_MIN_BLOCKS) k_compute(const LightParams P, uint32_t n, const int32_t *explicit_cubes) {
    __shared__ float s_lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    if (!explicit_cubes) n = P.scalars[0];   // the round's list
    unsigned long long total_visits = 0;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t width = batch_width(P, n, n_warps);
    // batches of `width` consecutive list entries, handed out by a counter: a warp whose cubes see open air walks
    // ten times the nodes of one whose cubes are enclosed
    for (;;) {
        uint32_t batch = 0;
        if (explicit_cubes) {
            batch = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // (one batch per warp: the grid covers n)
        } else {
            if (lane == 0) batch = atomicAdd(P.scalars + 7, 1u);
            batch = __shfl_sync(0xffffffffu, batch, 0);
        }
        const uint32_t base = batch * (explicit_cubes ? 32u : width);
        if (base >= n) break;
        const uint32_t i = base + lane;
        const bool active = i < n && (explicit_cubes || lane < width);
        int x = 0, y = 0, z = 0;
        if (active) {
            if (explicit_cubes) {
                x = explicit_cubes[3 * i]; y = explicit_cubes[3 * i + 1]; z = explicit_cubes[3 * i + 2];
            } else {
                cube_of(P.scene, P.list[i], x, y, z);
            }
        }
        uint32_t visits = 0;
        const uint32_t nv = compute_light_lockstep<false>(P, s_lut, active, x, y, z, 0, &visits);
        if (active) P.new_light[i] = nv;
        total_visits += visits;
        if (explicit_cubes) break;
    }
    for (int off = 16; off > 0; off >>= 1) total_visits += __shfl_down_sync(0xffffffffu, total_visits, off);
    if (lane == 0 && total_visits) atomicAdd(reinterpret_cast<unsigned long long *>(P.scalars + 4), total_visits);
}

// compute_light / the dependency re-queue with the chain walk (light_kernel.cuh: compute_light_chains): one warp per
// cube, cubes handed out by a counter.  k_walk_chains<false> writes new_light for the round's list (or explicit
// cubes); a cube one of whose chains needs more than LIGHT_CHAIN_K terms goes to the overflow list and is computed by
// the lockstep walk (k_compute_overflow).  k_walk_chains<true> is k_mark for the entries of `changed`.
template <bool MARK>
__global__ void __launch_bounds__(128, CHAIN_WALK_BLOCKS_PER_SM) k_walk_chains(const LightParams P, uint32_t n, const int32_t *explicit_cubes) {
    __shared__ float s_lut[256];
    __shared__ ChainShared s_sh[4];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    ChainShared &sh = s_sh[wib];
    float4 *terms = P.term_scratch + (size_t)(blockIdx.x * 4 + wib) * LIGHT_WARP_SCRATCH_F4;
    if (!explicit_cubes) n = MARK ? P.scalars[6] : P.scalars[0];
    unsigned long long total_visits = 0;
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(P.scalars + (MARK ? 8 : 7), 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= n) break;
        const uint32_t i = MARK ? P.changed[item] : item;   // position in the round's list
        int x, y, z;
        if (explicit_cubes) { x = explicit_cubes[3 * i]; y = explicit_cubes[3 * i + 1]; z = explicit_cubes[3 * i + 2]; }
        else cube_of(P.scene, P.list[i], x, y, z);
        const uint32_t prio = MARK ? (uint32_t)P.diff[i] / 2u + 1u : 0u;
        uint32_t visits = 0;
        bool overflowed = false;
        const uint32_t nv = compute_light_chains<MARK>(P, s_lut, sh, terms, x, y, z, prio, &visits, &overflowed);
        if (!MARK && lane == 0) {
            if (overflowed) P.overflow[atomicAdd(P.scalars + 9, 1u)] = i;
            else P.new_light[i] = nv;
        }
        total_visits += visits;
    }
    if (!MARK && lane == 0 && total_visits) atomicAdd(reinterpret_cast<unsigned long long *>(P.scalars + 4), total_visits);
}

// the cubes the chain walk could not hold (scalars[9] entries of `overflow`), by the lockstep walk
__global__ void __launch_bounds__(128, AICB_LIGHT_MIN_BLOCKS) k_compute_overflow(const LightParams P, const int32_t *explicit_cubes) {
    __shared__ float s_lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    const uint32_t n = P.scalars[9];
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
        const uint32_t nv = compute_light_lockstep<false>(P, s_lut, active, x, y, z, 0, &visits);
        if (active) P.new_light[i] = nv;
        total_visits += visits;
    }
    for (int off = 16; off > 0; off >>= 1) total_visits += __shfl_down_sync(0xffffffffu, total_visits, off);
    if (lane == 0 && total_visits) atomicAdd(reinterpret_cast<unsigned long long *>(P.scalars + 4), total_visits);
}

// apply_light_update (updater.rs:295-363) minus the dependency re-queue (k_mark)
__global__ void k_apply(const LightParams P) {
    const uint32_t n = P.scalars[0];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t idx = P.list[i];
    uint32_t *light = const_cast<uint32_t *>(P.scene.light);
    const uint32_t old = light[idx], nv = P.new_light[i];
    const int d = difference_priority(nv, old);
    P.diff[i] = (uint8_t)d;
    atomicAdd(P.scalars + 3, 1u);
    if (d > 0) {
        light[idx] = nv;
        atomicMax(P.scalars + 2, (uint32_t)d);
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
            atomicCAS(&light[nidx], nl, g);
        }
    }
    }
}

// apply_light_update re-queues a cube's dependencies only when its packed difference exceeds 1 (updater.rs:355-360).
// The entries of the round's list that did are compacted (in list order within a block of 256) so that the warps of
// k_mark walk the chart for 32 cubes that all need it.
__global__ void __launch_bounds__(256) k_compact_changed(const LightParams P) {
    __shared__ uint32_t s_part[8], s_base;
    const uint32_t n = P.scalars[0];
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
            s_base = total ? atomicAdd(P.scalars + 6, total) : 0u;
        }
        __syncthreads();
        if (keep) P.changed[s_base + s_part[wid] + inc - 1] = i;
        __syncthreads();
    }
}

// the dependency re-queue of apply_light_update (updater.rs:355-360): re-walk the chart, raising the
// queue priority of every cube whose light was read
__global__ void __launch_bounds__(128, AICB_LIGHT_MIN_BLOCKS) k_mark(const LightParams P) {
    const uint32_t n = P.scalars[6];   // entries of the round's list that changed by more than one unit
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t width = batch_width(P, n, n_warps);
    for (;;) {
        uint32_t batch = 0;
        if (lane == 0) batch = atomicAdd(P.scalars + 8, 1u);
        batch = __shfl_sync(0xffffffffu, batch, 0);
        const uint32_t base = batch * width;
        if (base >= n) break;
        const bool active = base + lane < n && lane < width;
        const uint32_t i = active ? P.changed[base + lane] : 0u;
        const int d = active ? (int)P.diff[i] : 0;
        int x = 0, y = 0, z = 0;
        if (active) cube_of(P.scene, P.list[i], x, y, z);
        compute_light_lockstep<true>(P, P.scene.tables, active, x, y, z, (uint32_t)(d / 2 + 1), nullptr);
    }
}

// fast_evaluate_light (updater.rs:537-582): one thread per (x, z) column, top down
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
        light[idx] = value;
        P.pending[idx] = pend;
    }
}

struct EditOp {
    uint32_t idx;
    uint32_t cell;        // new cell word, or 0xffffffff = leave
    uint8_t set_opaque;   // light := OPAQUE
    uint8_t pending_op;   // 0 none, 1 remove, 2 raise to NEWLY_VISIBLE
    uint8_t _pad[2];
};

__global__ void k_edits(const LightParams P, const EditOp *ops, uint32_t n, uint32_t wide) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const EditOp op = ops[i];
    if (op.cell != 0xffffffffu) {
        if (wide) ((uint32_t *)P.scene.cells)[op.idx] = op.cell;
        else ((uint16_t *)P.scene.cells)[op.idx] = (uint16_t)op.cell;
    }
    if (op.set_opaque) const_cast<uint32_t *>(P.scene.light)[op.idx] = TX_OPAQUE;
    if (op.pending_op == 1) P.pending[op.idx] = 0;
    else if (op.pending_op == 2) P.pending[op.idx] = PRIO_NEWLY_VISIBLE;
}

LightParams make_params(aicb_scene *s) {
    LightParams P;
    std::memset(&P, 0, sizeof P);
    P.scene = s->ds;
    P.blocks = s->d_light_blocks;
    P.chart = s->ctx->d_chart;
    P.chart_pre = s->ctx->d_chart_pre;
    P.sky_term = s->d_sky_term;
    P.chains = s->ctx->d_chains;
    P.node_rel = s->ctx->d_node_rel;
    P.euler = s->ctx->d_euler;
    P.n_chains = s->ctx->n_chains;
    P.n_euler = s->ctx->n_euler;
    P.term_scratch = s->ctx->d_term_scratch;
    P.overflow = s->d_changed;   // (k_compute's overflow list and k_mark's work list are never live together)
    P.chart_nodes = s->ctx->chart_nodes;
    P.tile_max = s->d_tile_max;
    P.changed = s->d_changed;
    P.pending = s->d_pending;
    P.list = s->d_list;
    P.new_light = s->d_new_light;
    P.diff = s->d_diff;
    P.scalars = s->d_scalars;
    P.volume = (uint32_t)s->volume;
    P.max_distance = s->light_max_distance;
    return P;
}

aicb_status ensure_light_state(aicb_scene *s) {
    if (s->light_max_distance == 0) return aicb_fail(AICB_ERR_INVALID, "scene has LightPhysics::None (light_max_distance == 0)");
    aicb_status st = ensure_chart(s->ctx);
    if (st != AICB_OK) return st;
    if (!s->d_light) {  // a scene created without a light volume starts all NO_RAYS (initialize_light, updater.rs:628-656)
        std::vector<uint32_t> init(s->volume, TX_NO_RAYS);
        CU(cudaMalloc(&s->d_light, s->volume * 4 + 16));
        CU(cudaMemcpy(s->d_light, init.data(), s->volume * 4, cudaMemcpyHostToDevice));
        s->ds.light = s->d_light;
        s->device_bytes += s->volume * 4;
    }
    if (!s->d_sky_term) {
        // end_of_ray (updater.rs:889-924) without the lane's alpha and bundle weight: per chart node, the sky light
        // its bundle collects — the same f32 operations, in the same order, as the reference evaluates per ray end
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
                const uint32_t tx = s->ds.sky_faces[f];
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
        CU(cudaMalloc(&s->d_sky_term, sky.size() * sizeof(float4)));
        CU(cudaMemcpy(s->d_sky_term, sky.data(), sky.size() * sizeof(float4), cudaMemcpyHostToDevice));
        s->device_bytes += sky.size() * sizeof(float4);
    }
    if (!s->d_pending) {
        CU(cudaMalloc(&s->d_pending, s->volume + 16));
        CU(cudaMemset(s->d_pending, 0, s->volume + 16));
        CU(cudaMalloc(&s->d_list, s->volume * 4 + 16));
        CU(cudaMalloc(&s->d_new_light, s->volume * 4 + 16));
        CU(cudaMalloc(&s->d_diff, s->volume + 16));
        CU(cudaMalloc(&s->d_scalars, 16 * 4));
        CU(cudaMalloc(&s->d_tile_max, ((s->volume + LIGHT_TILE - 1) / LIGHT_TILE + 1) * 4));
        CU(cudaMalloc(&s->d_changed, s->volume * 4 + 16));
        s->device_bytes += s->volume * 4;
        s->device_bytes += s->volume * 10;
    }
    return AICB_OK;
}

// AICB_LIGHT_WALK=lockstep selects the previous walk (32 cubes per warp in lockstep) for comparisons
bool use_chain_walk() {
    const char *e = getenv("AICB_LIGHT_WALK");
    return !(e && std::strcmp(e, "lockstep") == 0);
}

// evaluate_light (space.rs:1496-1527): rounds until the highest queued priority is <= from_difference(epsilon)
aicb_status propagate(aicb_scene *s, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff, uint64_t *node_visits) {
    aicb_ctx *ctx = s->ctx;
    cudaStream_t st = ctx->stream;
    LightParams P = make_params(s);
    P.epsilon_priority = (uint32_t)epsilon / 2 + 1;
    {
        // Cubes within 16 priority levels of the round's maximum are relaxed together: far fewer rounds than strict
        // level-by-level relaxation (few cubes per round leave the GPU idle) for 8 % more updates; the parity
        // contract (tests/test_gpu_light.py) holds for every band, 0 = one level per round, 255 = all pending cubes.
        const char *e = getenv("AICB_LIGHT_BAND");
        P.priority_band = e ? (uint32_t)atoi(e) : 16u;
        const char *w = getenv("AICB_LIGHT_WIDTH");        // experiments: a fixed batch width (1..32)
        P.batch_width = w ? (uint32_t)atoi(w) : 0u;
        const char *b = getenv("AICB_LIGHT_BATCHES_PER_WARP");
        P.batches_per_warp = b ? (uint32_t)atoi(b) : 2u;
        const char *m = getenv("AICB_LIGHT_MIN_WIDTH");
        P.min_batch_width = m ? (uint32_t)atoi(m) : 4u;
        if (P.batch_width > 32) P.batch_width = 32;
        if (P.batches_per_warp < 1) P.batches_per_warp = 1;
        if (P.min_batch_width < 1) P.min_batch_width = 1;
    }
    const int blocks = ctx->num_sms * 8;
    const int wide = ctx->num_sms * 8;    // 128-thread blocks of the lockstep kernels (one warp per 32 list entries, grid-stride)
    const uint32_t n_tiles = (uint32_t)((s->volume + LIGHT_TILE - 1) / LIGHT_TILE);
    uint64_t total = 0, visits = 0, rounds = 0;
    uint32_t maxd = 0;
    CU(cudaEventRecord(ctx->ev0, st));
    CU(cudaMemsetAsync(s->d_scalars, 0, 16 * 4, st));
    k_tile_rebuild<<<blocks, 256, 0, st>>>(P, n_tiles);   // (fast_evaluate / edits write the priority bytes directly)
    const int ROUNDS_PER_SYNC = 8;
    const bool chains = use_chain_walk();
    for (int batch = 0; batch < 100000; batch++) {
        for (int round = 0; round < ROUNDS_PER_SYNC; round++) {
            CU(cudaMemsetAsync(s->d_scalars, 0, 2 * 4, st));   // this round's count and priority
            CU(cudaMemsetAsync(s->d_scalars + 6, 0, 4 * 4, st));   // ... its count of changed cubes, the two work counters, the overflow count
            k_find_max<<<16, 256, 0, st>>>(P, n_tiles);
            k_gather<<<blocks, 256, 0, st>>>(P, n_tiles);
            if (chains) {
                k_walk_chains<false><<<ctx->chain_walk_blocks, 128, 0, st>>>(P, 0, nullptr);
                k_compute_overflow<<<wide, 128, 0, st>>>(P, nullptr);
            } else {
                k_compute<<<wide, 128, 0, st>>>(P, 0, nullptr);
            }
            k_apply<<<wide, 128, 0, st>>>(P);
            k_compact_changed<<<blocks, 256, 0, st>>>(P);
            if (chains) k_walk_chains<true><<<ctx->chain_walk_blocks, 128, 0, st>>>(P, 0, nullptr);
            else k_mark<<<wide, 128, 0, st>>>(P);
        }
        uint32_t h[8];
        CU(cudaMemcpyAsync(h, s->d_scalars, 8 * 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        CU(cudaGetLastError());
        if (getenv("AICB_LIGHT_TRACE"))
            fprintf(stderr, "[aicb200 light] batch %d: last round %u cubes at priority %u; %u updates so far\n", batch, h[0], h[1], h[3]);
        total = h[3];
        visits = (uint64_t)h[4] | ((uint64_t)h[5] << 32);
        maxd = h[2];
        rounds += ROUNDS_PER_SYNC;
        if (h[1] <= P.epsilon_priority) break;   // the batch's last round found nothing above epsilon
    }
    CU(cudaEventRecord(ctx->ev1, st));
    CU(cudaEventSynchronize(ctx->ev1));
    float ms = 0.0f;
    CU(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    s->light_stats[0] = total;
    s->light_stats[1] = visits;
    s->light_stats[2] = rounds;
    s->light_stats[3] = (uint64_t)(ms * 1000.0f);   // device time of the propagation in microseconds
    if (updates_done) *updates_done = total;
    if (max_diff) *max_diff = (uint8_t)maxd;
    if (node_visits) *node_visits = visits;
    return AICB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// called from aicb200.cu
// ---------------------------------------------------------------------------------------------
aicb_status aicb_light_scene_upload(aicb_scene *s, const aicb_scene_desc *d) {
    s->light_max_distance = d->light_max_distance;
    if (s->volume) s->h_ids.assign(d->block_ids, d->block_ids + s->volume);
    std::vector<LightBlockDev> lb(d->n_blocks);
    s->h_block_light.resize(d->n_blocks);
    for (size_t i = 0; i < d->n_blocks; i++) {
        const aicb_block_desc &b = d->blocks[i];
        LightBlockDev &o = lb[i];
        std::memcpy(o.face_color[0], b.light_color, 16);
        for (int f = 0; f < 6; f++) std::memcpy(o.face_color[f + 1], b.light_face_colors[f], 16);
        std::memcpy(o.emission, b.light_emission, 12);
        uint32_t fl = b.light_opaque_faces & 0x3f;
        if (fl == 0x3f) fl |= LB_ALL_OPAQUE;
        if (b.light_visible) fl |= LB_VISIBLE;
        if (!(b.light_emission[0] == 0.0f && b.light_emission[1] == 0.0f && b.light_emission[2] == 0.0f)) fl |= LB_EMISSIVE;
        o.flags = fl;
        s->h_block_light[i] = fl;
    }
    if (!lb.empty()) {
        CU(cudaMalloc(&s->d_light_blocks, lb.size() * sizeof(LightBlockDev)));
        CU(cudaMemcpy(s->d_light_blocks, lb.data(), lb.size() * sizeof(LightBlockDev), cudaMemcpyHostToDevice));
        s->device_bytes += lb.size() * sizeof(LightBlockDev);
    }
    return AICB_OK;
}

// the light-side records of replaced block definitions (aicb_scene_update_blocks)
aicb_status aicb_light_blocks_update(aicb_scene *s, const uint16_t *indices, const aicb_block_desc *descs, size_t n) {
    for (size_t i = 0; i < n; i++) {
        const aicb_block_desc &b = descs[i];
        LightBlockDev o;
        std::memset(&o, 0, sizeof o);
        std::memcpy(o.face_color[0], b.light_color, 16);
        for (int f = 0; f < 6; f++) std::memcpy(o.face_color[f + 1], b.light_face_colors[f], 16);
        std::memcpy(o.emission, b.light_emission, 12);
        uint32_t fl = b.light_opaque_faces & 0x3f;
        if (fl == 0x3f) fl |= LB_ALL_OPAQUE;
        if (b.light_visible) fl |= LB_VISIBLE;
        if (!(b.light_emission[0] == 0.0f && b.light_emission[1] == 0.0f && b.light_emission[2] == 0.0f)) fl |= LB_EMISSIVE;
        o.flags = fl;
        if (indices[i] < s->h_block_light.size()) s->h_block_light[indices[i]] = fl;
        if (s->d_light_blocks) CU(cudaMemcpy(s->d_light_blocks + indices[i], &o, sizeof o, cudaMemcpyHostToDevice));
    }
    return AICB_OK;
}

void aicb_light_scene_free(aicb_scene *s) {
    if (s->d_light_blocks) cudaFree(s->d_light_blocks);
    if (s->d_pending) cudaFree(s->d_pending);
    if (s->d_list) cudaFree(s->d_list);
    if (s->d_new_light) cudaFree(s->d_new_light);
    if (s->d_diff) cudaFree(s->d_diff);
    if (s->d_scalars) cudaFree(s->d_scalars);
    if (s->d_tile_max) cudaFree(s->d_tile_max);
    if (s->d_changed) cudaFree(s->d_changed);
    if (s->d_sky_term) cudaFree(s->d_sky_term);
}

void aicb_light_ctx_free(aicb_ctx *c) { free_chart(c); }

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
    if (!s) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    aicb_status st = ensure_light_state(s);
    if (st != AICB_OK) return st;
    LightParams P = make_params(s);
    const uint32_t cols = (uint32_t)s->ds.size[0] * (uint32_t)s->ds.size[2];
    if (cols) k_fast_evaluate<<<(cols + 127) / 128, 128, 0, s->ctx->stream>>>(P);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s->ctx->stream));
    return AICB_OK;
}

aicb_status aicb_light_compute(aicb_scene *s, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]) {
    if (!s || (n && (!cubes || !out))) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n > s->volume) return aicb_fail(AICB_ERR_INVALID, "more cubes than the Space holds");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    aicb_status st = ensure_light_state(s);
    if (st != AICB_OK) return st;
    if (!n) return AICB_OK;
    LightParams P = make_params(s);
    int32_t *d_cubes = nullptr;
    CU(cudaMalloc(&d_cubes, n * 12));
    CU(cudaMemcpy(d_cubes, cubes, n * 12, cudaMemcpyHostToDevice));
    cudaMemsetAsync(s->d_scalars, 0, 16 * 4, s->ctx->stream);
    if (use_chain_walk()) {
        k_walk_chains<false><<<s->ctx->chain_walk_blocks, 128, 0, s->ctx->stream>>>(P, (uint32_t)n, d_cubes);
        k_compute_overflow<<<s->ctx->num_sms * 8, 128, 0, s->ctx->stream>>>(P, d_cubes);
    } else {
        k_compute<<<(unsigned)((n + 127) / 128), 128, 0, s->ctx->stream>>>(P, (uint32_t)n, d_cubes);
    }
    uint32_t h[16];
    cudaError_t e = cudaMemcpyAsync(out, s->d_new_light, n * 4, cudaMemcpyDeviceToHost, s->ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, s->d_scalars, sizeof h, cudaMemcpyDeviceToHost, s->ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s->ctx->stream);
    if (e == cudaSuccess) {
        s->light_stats[0] = n;
        s->light_stats[1] = (uint64_t)h[4] | ((uint64_t)h[5] << 32);
        s->light_stats[2] = h[9];   // cubes that took the lockstep walk (a chain with more terms than its slots)
        s->light_stats[3] = 0;
    }
    cudaFree(d_cubes);
    if (e != cudaSuccess) return aicb_cuda_fail(e, "light compute");
    return AICB_OK;
}

aicb_status aicb_light_evaluate(aicb_scene *s, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                                uint64_t *node_visits) {
    if (!s) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    aicb_status st = ensure_light_state(s);
    if (st != AICB_OK) return st;
    return propagate(s, epsilon, updates_done, max_diff, node_visits);
}

// Mutation::set x n (space.rs:1346-1352 -> side_effects_of_set -> modified_cube_needs_update,
// updater.rs:135-173) applied in order on the host mirror, then evaluate_light(epsilon).
aicb_status aicb_light_edit_and_propagate(aicb_scene *s, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n_edits,
                                          uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff) {
    if (!s || (n_edits && (!cubes || !new_ids))) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    aicb_status st = ensure_light_state(s);
    if (st != AICB_OK) return st;
    const DeviceScene &ds = s->ds;
    auto index_of = [&](int x, int y, int z, uint32_t *idx) {
        uint32_t dx = (uint32_t)(x - ds.lo[0]), dy = (uint32_t)(y - ds.lo[1]), dz = (uint32_t)(z - ds.lo[2]);
        if (dx >= (uint32_t)ds.size[0] || dy >= (uint32_t)ds.size[1] || dz >= (uint32_t)ds.size[2]) return false;
        *idx = (dx * (uint32_t)ds.size[1] + dy) * (uint32_t)ds.size[2] + dz;
        return true;
    };
    std::unordered_map<uint32_t, EditOp> ops;
    auto op_of = [&](uint32_t idx) -> EditOp & {
        auto it = ops.find(idx);
        if (it == ops.end()) {
            EditOp o;
            std::memset(&o, 0, sizeof o);
            o.idx = idx;
            o.cell = 0xffffffffu;
            it = ops.emplace(idx, o).first;
        }
        return it->second;
    };
    // validate everything before the host mirror (or anything else) changes
    for (size_t i = 0; i < n_edits; i++) {
        uint32_t idx;
        if (!index_of(cubes[i][0], cubes[i][1], cubes[i][2], &idx)) return aicb_fail(AICB_ERR_INVALID, "cube out of bounds");
        if (new_ids[i] >= s->h_block_light.size()) return aicb_fail(AICB_ERR_INVALID, "block id out of range");
    }
    for (size_t i = 0; i < n_edits; i++) {
        uint32_t idx;
        index_of(cubes[i][0], cubes[i][1], cubes[i][2], &idx);
        if (s->h_ids[idx] == new_ids[i]) continue;  // Mutation::set of the same block changes nothing
        s->h_ids[idx] = new_ids[i];
        EditOp &o = op_of(idx);
        o.cell = ds.wide_cells ? (new_ids[i] | ((uint32_t)s->block_kind[new_ids[i]] << 16))
                               : (new_ids[i] | ((uint32_t)s->block_kind[new_ids[i]] << 14));
        const uint32_t fl = s->h_block_light[new_ids[i]];
        if ((fl & LB_ALL_OPAQUE) && !(fl & LB_EMISSIVE)) {  // opaque_for_light_computation
            o.set_opaque = 1;
            o.pending_op = 1;
        } else {
            o.pending_op = 2;
        }
        for (int f = 0; f < 6; f++) {
            const int sgn = (f < 3) ? -1 : 1, a = f % 3;
            uint32_t nidx;
            if (!index_of(cubes[i][0] + (a == 0 ? sgn : 0), cubes[i][1] + (a == 1 ? sgn : 0), cubes[i][2] + (a == 2 ? sgn : 0), &nidx))
                continue;
            const int opp = (f < 3) ? f + 3 : f - 3;
            if (!((s->h_block_light[s->h_ids[nidx]] >> opp) & 1u)) op_of(nidx).pending_op = 2;
        }
    }
    if (!ops.empty()) {
        std::vector<EditOp> flat;
        flat.reserve(ops.size());
        for (auto &kv : ops) flat.push_back(kv.second);
        EditOp *d_ops = nullptr;
        CU(cudaMalloc(&d_ops, flat.size() * sizeof(EditOp)));
        CU(cudaMemcpyAsync(d_ops, flat.data(), flat.size() * sizeof(EditOp), cudaMemcpyHostToDevice, s->ctx->stream));
        LightParams P = make_params(s);
        k_edits<<<(unsigned)((flat.size() + 127) / 128), 128, 0, s->ctx->stream>>>(P, d_ops, (uint32_t)flat.size(), ds.wide_cells);
        cudaError_t e = cudaStreamSynchronize(s->ctx->stream);
        cudaFree(d_ops);
        if (e != cudaSuccess) return aicb_cuda_fail(e, "light edits");
    }
    return propagate(s, epsilon, updates_done, max_diff, nullptr);
}

aicb_status aicb_light_download(aicb_scene *s, uint8_t (*out)[4], size_t n_texels) {
    if (!s || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if (n_texels != s->volume) return aicb_fail(AICB_ERR_INVALID, "light volume size mismatch");
    if (!s->d_light) return aicb_fail(AICB_ERR_INVALID, "scene has no light volume (LightPhysics::None)");
    std::lock_guard<std::mutex> lock(s->ctx->mu);
    CU(cudaSetDevice(s->ctx->device));
    // ordered behind everything queued on the context's stream (cube deltas, propagation)
    CU(cudaMemcpyAsync(out, s->d_light, s->volume * 4, cudaMemcpyDeviceToHost, s->ctx->stream));
    CU(cudaStreamSynchronize(s->ctx->stream));
    return AICB_OK;
}

aicb_status aicb_light_stats(const aicb_scene *s, uint64_t out[4]) {
    if (!s || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    for (int i = 0; i < 4; i++) out[i] = s->light_stats[i];
    return AICB_OK;
}
}
