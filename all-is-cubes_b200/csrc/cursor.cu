// cursor.cu — the cursor over a scene's cells on the device: cursor_raycast (all-is-cubes/src/character/cursor.rs:26-107)
// and StandardCameras::project_cursor (all-is-cubes-render/src/camera/stdcam.rs:357-389) for a batch of queries, on one
// context and on a device group.  One thread per query walks the Space level with the frames' Raycaster arithmetic
// (caster_begin / caster_step), reads each cube's block record, and for a recursive block walks its voxels with the
// same caster, until a cube is selectable.  The selectability bits live in words the table already had: BlockRec::flags
// and the .w lane of a palette entry's emission (block_words.cuh: voxel_flags).  A call reads the scene and writes
// only its results: the host mirror of the block ids, the light state and a frame in flight are left alone.
#include <cmath>
#include <vector>

#include "internal.h"

using namespace aicb;

namespace {

// One layer of a batch: the scene it walks, and for project_cursor its camera (its ray per NDC point), its maximum
// distance and the `layer` value a query it answers records.
struct CursorLayer {
    DeviceScene scene;
    double m[16];          // Camera::inverse_projection_view (ndc queries)
    double max_distance;   // without per-query distances
    uint32_t code;
    uint32_t wide_bricks;  // SpaceHost::wide_bricks: u32 brick words
};

struct CursorParams {
    CursorLayer layer[2];          // tried in this order
    uint32_t n_layers;
    const double *rays;            // [n][6] origin, direction; or nullptr: ndc
    const double *ndc;             // [n][2]
    const double *max_distance;    // [n], or nullptr: each layer's max_distance
    aicb_cursor *out;
    uint64_t n;
};

// Camera::project_ndc_into_world (camera_struct.rs:238-257) with plain IEEE divisions (aicb_camera_project_ndc).
__device__ void ndc_ray(const double *m, double x, double y, double o[3], double d[3]) {
    double p[2][3];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const double z = (double)k;
        const double hx = x * m[0] + y * m[4] + z * m[8] + m[12];
        const double hy = x * m[1] + y * m[5] + z * m[9] + m[13];
        const double hz = x * m[2] + y * m[6] + z * m[10] + m[14];
        const double hw = x * m[3] + y * m[7] + z * m[11] + m[15];
        if (hw > 0.0) {
            p[k][0] = hx / hw;
            p[k][1] = hy / hw;
            p[k][2] = hz / hw;
        } else {
            p[k][0] = p[k][1] = p[k][2] = __longlong_as_double(0x7ff8000000000000LL);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
        o[a] = p[0][a];
        d[a] = p[1][a] - p[0][a];
    }
}

__device__ __forceinline__ uint32_t word_bits(float w) { return __float_as_uint(w); }

// A cube's block id from its cell word.
__device__ __forceinline__ uint32_t cell_id(const DeviceScene &S, uint32_t idx) {
    return S.wide_cells ? (__ldg((const uint32_t *)S.cells + idx) & 0xffffu)
                        : ((uint32_t)__ldg((const uint16_t *)S.cells + idx) & 0x3fffu);
}

// A palette entry's AICB_VOXEL_NOT_SELECTABLE bit.
__device__ __forceinline__ bool entry_selectable(const DeviceScene &S, uint32_t entry) {
    return (word_bits(__ldg(&S.palette[2 * (size_t)entry + 1].w)) & AICB_VOXEL_NOT_SELECTABLE) == 0;
}

__device__ __forceinline__ uint32_t texel_at(const DeviceScene &S, uint32_t idx) {
    return S.light ? __ldg(S.light + idx) : TEXEL_ONE;
}

// cursor_raycast on one scene: true with *c written if a cube was selected.  `o`, `d_in`: the ray as given.
__device__ bool cursor_cast(const DeviceScene &S, bool wide_bricks, const double o[3], const double d_in[3],
                            double max_distance, aicb_cursor *c) {
    // ray.direction.normalize() (euclid: self / self.length())
    const double len = sqrt(d_in[0] * d_in[0] + d_in[1] * d_in[1] + d_in[2] * d_in[2]);
    double d[3] = {d_in[0] / len, d_in[1] / len, d_in[2] / len};
    // Parameters::new (raycast.rs:749-771)
    if (!((fabs(d[0]) < 1e100) & (fabs(d[1]) < 1e100) & (fabs(d[2]) < 1e100))) d[0] = d[1] = d[2] = 0.0;
    Ray r;
    r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
    r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    r.sx = signum_101(d[0]); r.sy = signum_101(d[1]); r.sz = signum_101(d[2]);
    r.tdx = 1.0 / fabs(d[0]); r.tdy = 1.0 / fabs(d[1]); r.tdz = 1.0 / fabs(d[2]);
    r.half_over_len = 0.5 / sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    Level lv;
    lv.lox = S.lo[0]; lv.loy = S.lo[1]; lv.loz = S.lo[2];
    lv.nx = S.size[0]; lv.ny = S.size[1]; lv.nz = S.size[2];
    lv.base = 0;
    Caster cs;
    bool valid;
    // .within(space.bounds(), false): the exit step is not a step of this cast
    if (!caster_begin(cs, r, o[0], o[1], o[2], lv, &valid)) return false;
    for (;;) {
        if (cs.last_t > max_distance) return false;
        const uint32_t id = cell_id(S, cs.idx);
        const uint4 *bp = reinterpret_cast<const uint4 *>(S.blocks + id);
        const uint4 b0 = __ldg(bp), b1 = __ldg(bp + 1);   // BlockRec: b1 = brick_off, pal_off, flags, _pad
        const int cube[3] = {cs.rx + S.lo[0], cs.ry + S.lo[1], cs.rz + S.lo[2]};
        int face_selected = -1;
        if (!(b1.z & AICB_BLOCK_NOT_SELECTABLE)) {
            if ((b0.x & 0xffu) != KIND_RECURSIVE) {   // Evoxels::single_voxel: the block's one palette entry
                if (entry_selectable(S, b1.y)) face_selected = cs.face;
            } else {
                // step.recursive_raycast(ray, resolution, voxel_bounds) (raycast.rs:458-476)
                const double fres = (double)(b0.x >> 8);
                Level in;
                in.lox = (int16_t)(b0.y & 0xffff); in.loy = (int16_t)(b0.y >> 16); in.loz = (int16_t)(b0.z & 0xffff);
                in.nx = (int)(b0.z >> 16); in.ny = (int)(b0.w & 0xffff); in.nz = (int)(b0.w >> 16);
                in.base = b1.x;
                Caster ic;
                bool ivalid;
                if (caster_begin(ic, r, (o[0] - (double)cube[0]) * fres, (o[1] - (double)cube[1]) * fres,
                                 (o[2] - (double)cube[2]) * fres, in, &ivalid)) {
                    const int first_face = ic.face;   // a face of voxel_bounds
                    for (;;) {
                        const uint32_t w = wide_bricks ? __ldg((const uint32_t *)S.bricks + ic.idx) >> 16
                                                             : (uint32_t)(__ldg(S.bricks + ic.idx) & 0x7fffu);
                        if (entry_selectable(S, b1.y + w)) {
                            face_selected = first_face;
                            break;
                        }
                        // the exit step's cube is outside voxel_bounds: get_opt_evoxel gives nothing
                        if (!ivalid || caster_step(ic, r, in.nx, in.ny, in.nz)) break;
                    }
                }
            }
        }
        if (face_selected >= 0) {
            const int face = cs.face;
            double p[3];
            const double tm[3] = {cs.tmx, cs.tmy, cs.tmz};
            const int sg[3] = {r.sx, r.sy, r.sz};
#pragma unroll
            for (int a = 0; a < 3; a++) {   // RaycastStep::intersection_point (raycast.rs:409-439)
                double q = (double)cube[a];
                if (face == AICB_FACE_WITHIN) {
                    q = o[a];
                } else if ((face - 1) % 3 == a) {
                    if (sg[a] < 0) q = q + 1.0;
                } else if (sg[a] == 0) {
                    q = o[a];
                } else {
                    const double off = (tm[a] - cs.last_t) * d[a];
                    q = q + (sg[a] > 0 ? (1.0 - rclamp01(off)) : rclamp01(-off));
                }
                p[a] = q;
            }
            int pc[3] = {cube[0], cube[1], cube[2]};
            if (face != AICB_FACE_WITHIN) pc[(face - 1) % 3] += face >= AICB_FACE_PX ? 1 : -1;   // cube_behind
            uint32_t pid = AICB_CURSOR_NONE, plight = 0;
            if (face != AICB_FACE_WITHIN) {
                const uint32_t dx = (uint32_t)(pc[0] - S.lo[0]), dy = (uint32_t)(pc[1] - S.lo[1]),
                               dz = (uint32_t)(pc[2] - S.lo[2]);
                if ((dx < (uint32_t)S.size[0]) & (dy < (uint32_t)S.size[1]) & (dz < (uint32_t)S.size[2])) {
                    const uint32_t pidx = (dx * (uint32_t)S.size[1] + dy) * (uint32_t)S.size[2] + dz;
                    pid = cell_id(S, pidx);
                    plight = texel_at(S, pidx);
                } else {
                    pid = AICB_CURSOR_OUTSIDE;
                    plight = S.light ? light_outside(S, pc[0], pc[1], pc[2]) : TEXEL_ONE;
                }
            }
            const uint32_t light = texel_at(S, cs.idx);
#pragma unroll
            for (int a = 0; a < 3; a++) {
                c->point_entered[a] = p[a];
                c->cube[a] = cube[a];
                c->preceding_cube[a] = pc[a];
            }
            c->distance = cs.last_t > 0.0 ? cs.last_t : 0.0;   // PositiveSign::new_clamped
            c->block_id = id;
            c->preceding_block_id = pid;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                c->light[k] = (uint8_t)(light >> (8 * k));
                c->preceding_light[k] = (uint8_t)(plight >> (8 * k));
            }
            c->face_entered = (uint8_t)face;
            c->face_selected = (uint8_t)face_selected;
            return true;
        }
        if (!valid || caster_step(cs, r, lv.nx, lv.ny, lv.nz)) return false;
    }
}

__global__ void __launch_bounds__(128) cursor_kernel(const __grid_constant__ CursorParams P) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    aicb_cursor c;
    memset(&c, 0, sizeof c);
    c.block_id = c.preceding_block_id = AICB_CURSOR_NONE;
    for (uint32_t k = 0; k < P.n_layers; k++) {
        const CursorLayer &L = P.layer[k];
        double o[3], d[3];
        if (P.rays) {
#pragma unroll
            for (int a = 0; a < 3; a++) {
                o[a] = P.rays[6 * i + a];
                d[a] = P.rays[6 * i + 3 + a];
            }
        } else {
            ndc_ray(L.m, P.ndc[2 * i], P.ndc[2 * i + 1], o, d);
        }
        const double max_distance = P.max_distance ? P.max_distance[i] : L.max_distance;
        if (cursor_cast(L.scene, L.wide_bricks != 0, o, d, max_distance, &c)) {
            c.layer = (uint8_t)L.code;
            break;
        }
    }
    P.out[i] = c;
}

// One layer as the host gives it: each replica's scene, and for project_cursor its camera.
struct LayerArg {
    aicb_scene *const *scene;
    const aicb_camera *camera;
    double max_distance;
    uint32_t code;
};

// The batch (in device 0's memory) cut into ranges of whole warps, one per listed context as aicb_group_trace_rays
// cuts its rays; context i walks its own replica and stores into device 0's `out`.  Device 0's stream ends after every
// part (fan_in), and device 0 is current.
aicb_status issue_cursor(aicb_ctx *const *ctx, size_t n_ctx, const LayerArg *layers, uint32_t n_layers,
                         const double *rays, const double *ndc, const double *max_distance, aicb_cursor *out, size_t n) {
    const std::vector<WarpRange> ranges = warp_ranges(n, n_ctx);
    TRY(fan_out(ctx, ranges.size()));
    for (size_t i = 0; i < ranges.size(); i++) {
        const size_t begin = ranges[i].begin, count = ranges[i].count;
        if (count == 0) continue;
        CursorParams P;
        memset(&P, 0, sizeof P);
        P.n_layers = n_layers;
        for (uint32_t k = 0; k < n_layers; k++) {
            const aicb_scene *s = layers[k].scene[i];
            P.layer[k].scene = s->ds;
            if (layers[k].camera) memcpy(P.layer[k].m, layers[k].camera->inverse_projection_view, sizeof P.layer[k].m);
            P.layer[k].max_distance = layers[k].max_distance;
            P.layer[k].code = layers[k].code;
            P.layer[k].wide_bricks = s->host->wide_bricks ? 1u : 0u;
        }
        P.rays = rays ? rays + 6 * begin : nullptr;
        P.ndc = ndc ? ndc + 2 * begin : nullptr;
        P.max_distance = max_distance ? max_distance + begin : nullptr;
        P.out = out + begin;
        P.n = count;
        CU(cudaSetDevice(ctx[i]->device));
        cursor_kernel<<<(unsigned)((count + 127) / 128), 128, 0, ctx[i]->stream.get()>>>(P);
        CU(cudaGetLastError());
    }
    return fan_in(ctx, ranges.size());
}

// The host form: the queries staged in device 0's d_cursor, the results copied back once every part is done.
aicb_status cursor_host(aicb_ctx *const *ctx, size_t n_ctx, const LayerArg *layers, uint32_t n_layers,
                        const double *rays, const double *ndc, const double *max_distance, aicb_cursor *out, size_t n) {
    aicb_ctx *c0 = ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n == 0) return AICB_OK;
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t in_bytes = n * (rays ? 6 : 2) * sizeof(double);
    const size_t out_at = 0, in_at = up(n * sizeof(aicb_cursor)), md_at = in_at + up(in_bytes);
    TRY(c0->d_cursor.ensure(md_at + (max_distance ? n * sizeof(double) : 0)));
    char *base = c0->d_cursor.get<char>();
    cudaStream_t s = c0->stream.get();
    CU(cudaMemcpyAsync(base + in_at, rays ? (const void *)rays : (const void *)ndc, in_bytes, cudaMemcpyHostToDevice, s));
    if (max_distance) CU(cudaMemcpyAsync(base + md_at, max_distance, n * sizeof(double), cudaMemcpyHostToDevice, s));
    const double *d_in = reinterpret_cast<const double *>(base + in_at);
    TRY(issue_cursor(ctx, n_ctx, layers, n_layers, rays ? d_in : nullptr, rays ? nullptr : d_in,
                     max_distance ? reinterpret_cast<const double *>(base + md_at) : nullptr,
                     reinterpret_cast<aicb_cursor *>(base + out_at), n));
    CU(cudaMemcpyAsync(out, base + out_at, n * sizeof(aicb_cursor), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return AICB_OK;
}

aicb_status raycast_host(Replicas r, const double (*origin_dir)[6], const double *max_distance, size_t n,
                         aicb_cursor *out) {
    if (n && (!origin_dir || !out)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    const LayerArg layer = {r.scene, nullptr, HUGE_VAL, 0};
    return cursor_host(r.ctx, r.n, &layer, 1, &origin_dir[0][0], nullptr, max_distance, out, n);
}

aicb_status raycast_device(Replicas r, const double (*origin_dir)[6], const double *max_distance, size_t n,
                           aicb_cursor *out, cudaStream_t caller) {
    aicb_ctx *c0 = r.ctx[0];
    CU(cudaSetDevice(c0->device));
    if (n == 0) return AICB_OK;
    if (!origin_dir || !out) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    TRY(check_device_pointer(origin_dir, c0->device, false, 8, "origin_dir"));
    if (max_distance) TRY(check_device_pointer(max_distance, c0->device, false, 8, "max_distance"));
    TRY(check_device_pointer(out, c0->device, false, 8, "out"));
    TRY(join_caller(r.ctx, r.n, caller));
    const LayerArg layer = {r.scene, nullptr, HUGE_VAL, 0};
    TRY(issue_cursor(r.ctx, r.n, &layer, 1, &origin_dir[0][0], nullptr, max_distance, out, n));
    if (r.n > 1) CU(cudaStreamSynchronize(c0->stream.get()));   // a group call returns with its output final
    return release_caller(c0, caller);
}

// project_cursor's layers, UI first: each layer's scene on every listed context (`ui`, `world`: nullptr if absent).
aicb_status project_host(aicb_ctx *const *ctx, size_t n_ctx, aicb_scene *const *world, const aicb_camera *world_cam,
                         aicb_scene *const *ui, const aicb_camera *ui_cam, const double (*ndc)[2], size_t n,
                         double world_max_distance, aicb_cursor *out) {
    LayerArg layers[2];
    uint32_t k = 0;
    if (ui) layers[k++] = {ui, ui_cam, HUGE_VAL, 1};
    if (world) layers[k++] = {world, world_cam, world_max_distance, 2};
    return cursor_host(ctx, n_ctx, layers, k, nullptr, &ndc[0][0], nullptr, out, n);
}

aicb_status check_project(const void *world_scene, const aicb_camera *world_cam, bool world, const void *ui_scene,
                          const aicb_camera *ui_cam, bool ui, const double (*ndc)[2], size_t n, aicb_cursor *out) {
    if (n && (!ndc || !out)) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    if ((world && (!world_scene || !world_cam)) || (ui && (!ui_scene || !ui_cam)))
        return aicb_fail(AICB_ERR_INVALID, "a layer needs a scene and a camera");
    return AICB_OK;
}

}  // namespace

extern "C" {

aicb_status aicb_cursor_raycast(aicb_scene *s, const double (*origin_dir)[6], const double *max_distance, size_t n,
                                aicb_cursor *out) {
    return on_scene(s, [&](Replicas r) { return raycast_host(r, origin_dir, max_distance, n, out); });
}

aicb_status aicb_cursor_raycast_device(aicb_scene *s, const double (*origin_dir)[6], const double *max_distance,
                                       size_t n, aicb_cursor *out, void *stream) {
    return on_scene(s, [&](Replicas r) {
        return raycast_device(r, origin_dir, max_distance, n, out, (cudaStream_t)stream);
    });
}

aicb_status aicb_project_cursor(const aicb_layer *world, const aicb_layer *ui, const double (*ndc)[2], size_t n,
                                double world_max_distance, aicb_cursor *out) {
    TRY(check_project(world ? world->scene : nullptr, world ? world->camera : nullptr, world != nullptr,
                      ui ? ui->scene : nullptr, ui ? ui->camera : nullptr, ui != nullptr, ndc, n, out));
    if (world && ui && world->scene->ctx != ui->scene->ctx)
        return aicb_fail(AICB_ERR_INVALID, "the layers must be scenes of one context");
    if (!world && !ui) {
        for (size_t i = 0; i < n; i++) {
            memset(out + i, 0, sizeof *out);
            out[i].block_id = out[i].preceding_block_id = AICB_CURSOR_NONE;
        }
        return AICB_OK;
    }
    aicb_ctx *ctx = (world ? world->scene : ui->scene)->ctx;
    std::lock_guard<std::mutex> lock(ctx->mu);
    aicb_scene *ws = world ? world->scene : nullptr, *us = ui ? ui->scene : nullptr;
    return project_host(&ctx, 1, world ? &ws : nullptr, world ? world->camera : nullptr, ui ? &us : nullptr,
                        ui ? ui->camera : nullptr, ndc, n, world_max_distance, out);
}

aicb_status aicb_group_cursor_raycast(aicb_group_scene *gs, const double (*origin_dir)[6], const double *max_distance,
                                      size_t n, aicb_cursor *out) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return raycast_host(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, origin_dir, max_distance,
                        n, out);
}

aicb_status aicb_group_cursor_raycast_device(aicb_group_scene *gs, const double (*origin_dir)[6],
                                             const double *max_distance, size_t n, aicb_cursor *out, void *stream) {
    if (!gs) return aicb_fail(AICB_ERR_INVALID, "NULL argument");
    ContextLocks lock(gs->group->ctx);
    return raycast_device(Replicas{gs->scene.data(), gs->group->ctx.data(), gs->scene.size()}, origin_dir,
                          max_distance, n, out, (cudaStream_t)stream);
}

aicb_status aicb_group_project_cursor(const aicb_group_layer *world, const aicb_group_layer *ui, const double (*ndc)[2],
                                      size_t n, double world_max_distance, aicb_cursor *out) {
    TRY(check_project(world ? world->scene : nullptr, world ? world->camera : nullptr, world != nullptr,
                      ui ? ui->scene : nullptr, ui ? ui->camera : nullptr, ui != nullptr, ndc, n, out));
    if (world && ui && world->scene->group != ui->scene->group)
        return aicb_fail(AICB_ERR_INVALID, "the layers must be scenes of the same group");
    if (!world && !ui) return aicb_project_cursor(nullptr, nullptr, ndc, n, world_max_distance, out);
    aicb_group *g = (world ? world->scene : ui->scene)->group;
    ContextLocks lock(g->ctx);
    return project_host(g->ctx.data(), g->ctx.size(), world ? world->scene->scene.data() : nullptr,
                        world ? world->camera : nullptr, ui ? ui->scene->scene.data() : nullptr,
                        ui ? ui->camera : nullptr, ndc, n, world_max_distance, out);
}

}  // extern "C"
