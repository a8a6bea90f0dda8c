// trace_kernel.cuh — the device code of libaicb200's raytracer: a from-scratch sm_90a implementation of
// all-is-cubes' SpaceRaytracer::trace_ray (sr.rs:135-238) and its pixel dispatch (renderer.rs:424-451, 516-556).
//
// Design (GPU-first, not a translation).  One frame = three or four kernels on one stream:
//  * gen_kernel (one thread per ray, convergent): pixel -> world ray, Raycaster::new().within(space bounds); rays that
//    miss the space are finished here, the others are listed by chord length (longest first);
//  * trace_kernel (persistent warps): every lane owns one ray at a time and takes the next one from the list when it
//    finishes.  The hot loop does, for every lane, ONE Amanatides–Woo DDA step in f64 (select-based, branch-free), one
//    dependent 2-byte load, the step count / opacity test, and — predicated, in the same iteration — the two cheap
//    things a ray can meet: the end of a Volumetric span (an 8-byte store into the pending hit record) and a visible
//    surface (a 64-byte hit record written to the lane's own chunk of the hit stream).  Only a change of level
//    (entering a recursive block: Raycaster::within on the brick; leaving one) and the end of a ray park the lane; the
//    warp serves parked lanes together once enough of them wait.  The kernel evaluates no colour: of the transmittance
//    it keeps only an upper bound, in the log domain (one multiply-add per span), to know when the ray is certainly
//    opaque;
//  * shading (shade_hit), one thread per hit record, convergent: cube / voxel coordinates and the intersection point
//    from the recorded caster state, apply_transmittance (f64 pow), fog (f64 exp), the invisibility test and
//    compute_illumination;
//  * compositing, one thread per ray: the exact transmittance chain in ray order, the opacity cut; then per pixel the
//    sky, tone mapping, sRGB8 (finish_pixel).
//  With None / Flat lighting both happen in resolve_kernel (one warp per 8x4 tile of rays, the shaded hits in shared
//  memory) unless the previous frame was deep (launch_trace); otherwise in shade_kernel, then encode_kernel, through a
//  ShadedHit stream.
//  The kernels of a frame follow each other with programmatic dependent launch (grid_dependency_sync).  A frame with
//  LightingOption::Bounce runs shade + encode a second time per sample for the secondary rays (see the bounce_*
//  kernels).
//  The two-level grid (Space cubes -> block id; block -> N^3 brick of palette indices) is walked by ONE unified DDA;
//  entering a recursive block pushes the outer state (shared memory) and re-initialises the same DDA on the brick.
//  Cell words carry their classification in the top bits (bit 15 = nothing to see, on both levels).
//  All ray geometry is f64 and all colour is f32, operation for operation as the reference (compiled with
//  -fmad=false: Rust never contracts to FMA); powf/expf are evaluated in f64 and rounded once; the sRGB8 encode is a
//  search in a 255-entry threshold table built on the host with the platform powf.
//
// Every function cites the reference lines it reproduces.
#pragma once
#include <cstdint>
#include <type_traits>
#include <cuda_runtime.h>

#include "../../include/aicb200.h"

#ifdef __CUDACC__
#include <cuda_fp16.h>
#include "exact_math.cuh"
#endif

// The EvaluatedBlock members light reads (evaluated.rs:189-272), 128 bytes: light propagation's per-block record
// (light_kernel.cuh), here so that the host code that builds a scene's block table sees it too.
struct LightBlockDev {
    float face_color[7][4];  // Within, NX..PZ (face7_color)
    float emission[3];
    uint32_t flags;          // bits 0-5 opaque[NX..PZ], 6 all opaque, 7 visible_or_animated, 8 emission != 0
};
static_assert(sizeof(LightBlockDev) == 128, "LightBlockDev must be 128 bytes");

namespace aicb {

// ---- device-side scene -------------------------------------------------------------------------
// The kind sits in the top two bits of a u16 cell so that bit 15 means "nothing to see here" on both levels
// (brick words carry the same flag): the marching loop tests one bit.
// A brick word is a voxel's palette index (from its block's pal_off) with that flag, in one of two forms per scene:
// narrow, u16 = index | invisible<<15, while every palette has at most 32768 entries; wide, u32 = index<<16 |
// invisible<<15, for palettes of up to 65536 entries (VoxelIndex is u16).  trace_kernel's BRICK_WIDE reads the wide form.
constexpr uint32_t KIND_SINGLE = 0;     // Evoxels::One, visible
constexpr uint32_t KIND_RECURSIVE = 1;  // paletted brick
constexpr uint32_t KIND_INVISIBLE = 2;  // AIR, or a single voxel that is fully transparent + non-emissive

// 32-byte block record, read as two uint4.
struct BlockRec {
    uint32_t kind_res;     // kind | resolution << 8
    int16_t vlo[3];        // voxel_bounds lower
    uint16_t vsize[3];     // voxel_bounds size
    uint32_t brick_off;    // first u16 of this block's brick in the pool
    uint32_t pal_off;      // first palette entry (single: the voxel)
    uint32_t _pad[2];
};
static_assert(sizeof(BlockRec) == 32, "BlockRec must be 32 bytes");

struct DeviceScene {
    int32_t lo[3];
    int32_t size[3];
    const void *cells;          // u16 (id | kind<<14) or u32 (id | kind<<16), Z-major
    const uint32_t *light;      // PackedLight texels r|g<<8|b<<16|status<<24, or nullptr (== ONE)
    const BlockRec *blocks;
    const uint16_t *bricks;     // brick words: palette index | invisible<<15, or (wide pool) u32 index<<16 | invisible<<15
    const float4 *palette;      // 2 x float4 per entry: rgba, emission
    const float4 *blk_tab;      // per block id (single-voxel blocks): {alpha, upper bound of log2(1 - alpha), palette entry (bits), -}
    const float2 *pal_tab;      // per palette entry: {alpha, log2 bound} (what the marching kernel needs of a surface)
    const float *tables;        // [0,256): PackedLight decode LUT (data.rs:301-354); [256,512): sRGB8 thresholds;
                                // [512,768): PackedLight quantiser thresholds (light kernels)
    uint32_t sky_faces[6];      // BlockSky faces NX..PZ as texels (sky.rs:54-82)
    uint32_t sky_mean;
    uint32_t sky_kind;
    float sky_colors[8][3];
    uint32_t wide_cells;        // 0: u16 cells, 1: u32 cells
};

// One primary ray that enters the Space, after trace_ray_impl's prologue (sr.rs:135-180) and Raycaster::new().within()
// (raycast.rs:196-230): everything the marching kernel needs, in two arrays split by reader.  gen_kernel gives the
// rays it lists consecutive record indices (one atomic per warp), so a warp writes whole lines of both arrays.  The
// binned ray list and the hit records (HitRecord::task) hold the record index; the ray's task is in RayRecordB.
// A: what shading reads of a ray, one aligned half-line (4 x 16-byte loads); the marcher reads it too.
struct __align__(64) RayRecordA {
    double ox, oy, oz, dx, dy, dz;   // ray (direction already zeroed if |d| >= 1e100, raycast.rs:760-764)
    float t_to_view;                 // sr.rs:149-151
    uint32_t flags;                  // face | running<<3 | valid<<4 | active<<5 | (sx+1)<<6 | (sy+1)<<8 | (sz+1)<<10 | sky octant<<12
    double t_to_abs;                 // |d| of the original direction (sr.rs:146)
};
static_assert(sizeof(RayRecordA) == 64, "RayRecordA must be 64 bytes");
// B: what only the marcher reads, 5 x 16-byte loads.
struct __align__(16) RayRecordB {
    double tdx, tdy, tdz;            // t_delta
    double half_over_len;
    double tmx, tmy, tmz, last_t;    // outer caster at its first in-bounds cube
    int rx, ry, rz;                  // ... relative to the Space's lower corner (its index is (rx * ny + ry) * nz + rz)
    uint32_t task;                   // the ray's task in the chunk
};
static_assert(sizeof(RayRecordB) == 80, "RayRecordB must be 80 bytes");

// One surface of one ray, emitted by the marching kernel and lit by shade_hit: 64 bytes = 4 x 16-byte stores.
// It is the caster's state at the surface, not a derived geometry: cube / voxel coordinates, the intersection point
// (raycast.rs:409-439) and the palette entry are recovered from it by shade_hit, convergently.  The marcher
// evaluates no colour or transmittance: apply_transmittance (f64 pow), the fog amount (f64 exp), the invisibility
// test and the illumination all happen in shade_hit, and the transmittance chain of the ray is multiplied up in
// order by resolve_kernel or encode_kernel.
struct __align__(16) HitRecord {
    double tmx, tmy, tmz;   // State::t_max of the level the surface is on (unscaled)
    double last_t;          // State::last_t_distance of that level: Hit::t_distance = last_t / resolution
    uint32_t pal;           // palette entry (global index)
    uint32_t cell;          // linear index of the Space cube
    uint32_t vidx;          // inner level: index of the voxel in the brick pool
    uint32_t flags;         // face | inner<<3 | log2(resolution)<<4
    float thickness;        // Volumetric: length of the span inside the surface's material (world units); the record
                            // is written when the span closes; Surface / Threshold: 0; < 0: an unused slot (the tail of
                            // a lane's last chunk)
    uint32_t steps;         // the ray's step counter when the surface was shaded (the reference stops at the first
                            // counted step after the hit that brings the transmittance under 1/256; compositing
                            // needs the counter to restore that when the marcher's bound let the ray run on)
    uint32_t task;          // the ray: index of its RayRecordA / RayRecordB
    uint32_t next;          // in the last slot of a chunk: where the ray's hits continue (the first slot of another chunk)
};
static_assert(sizeof(HitRecord) == 64, "HitRecord must be 64 bytes");

// What shading yields per hit; shade_kernel leaves it in global memory for encode_kernel (one 32-byte sector).
struct __align__(32) ShadedHit {
    float r, g, b;       // outgoing light of the surface
    float factor;        // what it multiplies the ray's transmittance by (< 0: surface invisible / never shaded, skip)
    uint32_t next;
    uint32_t steps;
    uint32_t _pad[2];
};
static_assert(sizeof(ShadedHit) == 32, "ShadedHit must be 32 bytes");

// What the marching kernel hands to the resolve / encode kernel per ray (16 bytes).
struct __align__(16) TaskOut {
    uint32_t first_hit;  // index of the first HitRecord or 0xffffffff
    uint32_t steps;      // steps counted by the marcher (>= the reference's; see HitRecord::steps)
    uint32_t flags;      // sky octant
    uint32_t n_hits;     // hit records of this ray (consecutive slots; the last slot of a chunk links to the next chunk)
};

// Where a frame's kernels store their outputs, and what the layers hand on between passes (TraceParams::target).
struct TargetParams {
    uchar4 *out_srgb8;
    float4 *out_colorbuf;
    uint2 *out_rgba16f;         // premultiplied RGBA, 4 x f16 (raytrace_to_texture.rs:645-661)
    double *out_depth;
    aicb_hit *out_hit;
    uint32_t *out_steps;
    int32_t *out_text;          // CharacterBuf (text.rs:52-123) per pixel: block index of the first hit, or AICB_TEXT_*
    // layers (RtScene::trace_ray_through_layers, renderer.rs:454-478): a ray's accumulator can start from what the
    // layer in front left in it, and can be handed on instead of becoming a pixel
    const float4 *in_accum;     // per task (global index): ColorBuf (light, transmittance) to start from, or nullptr
    float4 *out_accum;          // per task: the ray's ColorBuf goes here and no pixel is produced, or nullptr
    float backdrop[4];          // Exception::Backdrop hit added after the ray (premultiplied light rgb, transmittance)
    uint32_t has_backdrop;
    float no_world[4];          // ColorBuf the accumulator is replaced by if it is not opaque in the end
    uint32_t has_no_world;
    // RaytraceToTexture's colour and depth targets (raytrace_to_texture.rs:591-683): read only by the TGT_TEX
    // instantiations of resolve_kernel / encode_kernel, and (the pixel list) by gen_kernel
    const uint32_t *pixel_list; // pixel task i is the framebuffer pixel pixel_list[i] = y * fb_width + x, or nullptr
    uint32_t n_list;
    uint32_t tex_layer;         // InLayer of this pass's hits: TEX_WORLD or TEX_UI (also the TGT_TERM text's layer)
    // A frame has one target, so the fields of the other target share the space: the parameter block, and with it
    // the code of the kernels that read neither, keeps its size.
    union {
        struct {
            float tex_exposure[2];      // exposure of the world and of the UI camera
            double depth_m[8];          // m13 m23 m33 m43 m14 m24 m34 m44 of the depth transform
            const double *in_depth;     // per task (global index): DepthBuf the layer in front left, or nullptr
            double *out_task_depth;     // per task: the ray's DepthBuf, handed on next to out_accum, or nullptr
            float *out_tex_depth;       // per pixel: the depth texel
        };
        // The terminal's ColorCharacterBuf (aicb_render_layers_terminal): read only by the TGT_TERM instantiations.
        // A CharacterBuf is (text, layer): an AICB_TEXT_* state or block index, and the tex_layer of the pass whose
        // Space the index belongs to.
        struct {
            aicb_terminal_pixel *out_term;  // per pixel: post-processed colour, text, layer
            const int2 *in_text;            // per task (global index): CharacterBuf the layer in front left, or nullptr
            int2 *out_task_text;            // per task: the ray's CharacterBuf, handed on next to out_accum, or nullptr
            int32_t text_start;             // CharacterBuf of a ray without in_text: Empty, or Hit(" ") behind a lone
                                            // backdrop
        };
    };
};

struct TraceParams {
    DeviceScene scene;
    // camera
    double m[16];               // inverse_projection_view, row-major m11..m44
    uint32_t fb_width, fb_height;
    double inv_width, inv_height;   // RN(1 / fb_width), RN(1 / fb_height): the pixel quotients by div_known_recip
    float exposure;
    // options
    uint32_t fog;
    uint32_t lighting;
    uint32_t transparency;
    float threshold;
    uint32_t antialias;
    uint32_t tone_mapping;
    float maximum_intensity;
    double view_distance;
    uint32_t debug_pixel_cost;
    uint32_t include_sky;
    // work description
    uint32_t local_rows;        // rows rendered by this shard
    uint32_t strip_rows, shard_index, shard_count;
    const double *rays;         // explicit rays (trace_rays) or nullptr (camera rays)
    uint64_t n_rays;            // number of explicit rays
    uint32_t tiles_x, tiles_y;
    uint32_t n_tasks;           // tiles_x * tiles_y * 32 (camera) or n_rays
    uint32_t out_full_frame;    // 1: outputs are indexed by framebuffer position (full-frame buffer, possibly peer memory)
    uint32_t n_samples;         // rays per pixel task: 4 with AntialiasingOption::Always, else 1
    uint32_t task_base;         // first task of the chunk being processed (tasks = pixel_task * n_samples + sample)
    // per-task streams between the kernels of a frame (HBM)
    RayRecordA *rays_a;         // gen -> march, shade (by record index)
    RayRecordB *rays_b;         // gen -> march
    unsigned int *ray_counter;  // records handed out in this chunk
    uint32_t *ray_index;        // per task: its record index (written for listed rays when non-null; the bounce kernels)
    TaskOut *task_out;          // march -> resolve / encode
    HitRecord *hits;            // march -> resolve / shade
    ShadedHit *shaded;          // shade -> encode (nullptr in a frame that runs resolve_kernel)
    unsigned int *hit_counter;  // hit slots handed out in this chunk (in chunks of HIT_CHUNK per lane)
    uint32_t *bin_list;         // gen -> march: record indices of the rays that enter the space, binned by chord length
    unsigned int *bin_count;    // [N_BINS] entries of each bin
    uint32_t bin_stride;        // capacity of one bin's list
    unsigned int *overflow_flag; // set when a chunk produced more hits than hit_capacity (frame must be re-run)
    uint32_t hit_capacity;
    uint32_t event_threshold;   // leave the marching loop once this many lanes wait (parked at a level switch, finished, idle)
    uint32_t tail_divisor;      // once the ray list is exhausted: leave the loop when (lanes that still have a ray) / this wait
    uint32_t refill_threshold;  // tail mode: once the ray list is exhausted and at most this many lanes of a warp still march,
                                // they run the lean per-lane loop
    TargetParams target;        // outputs
    // LightingOption::Bounce (surface.rs:113-166): the frame's primary pass and its secondary passes share these
    uint32_t bounce_mode;       // BOUNCE_OFF / BOUNCE_PRIMARY / BOUNCE_SECONDARY
    uint32_t bounce_samples;    // LightingOption::Bounce { samples }
    uint32_t bounce_pass;       // index of the secondary pass (sample) being traced
    uint32_t *bounce_req;       // per task of the chunk: slot of the fully opaque hit the ray ends on, or HIT_NONE
    unsigned long long *bounce_rng;  // per task: xoshiro256++ state (4 words)
    float4 *bounce_sum;         // per task: sum of the secondary rays' Rgb so far; .w = their cubes_traced (as bits)
    double *bounce_rays;        // per task: the secondary ray of this pass (origin, direction)
    unsigned long long *counters;  // [0] cubes_traced, [1] outer steps, [2] inner steps, [3] hits, [4] light texels, [5] blocks entered
    unsigned int *task_counter;
    unsigned long long *debug_warp_times;  // AICB_PROFILE_KERNELS: per marching warp {start ns, end ns, passes, rays}
};

#ifdef __CUDACC__

#define AICB_DEV __device__ __forceinline__
#define AICB_NOINLINE static __device__ __noinline__

constexpr int LC_NONE = 0, LC_FLAT = 1, LC_INTERP = 2, LC_BOUNCE = 3;  // lighting class (template)
constexpr uint32_t BOUNCE_OFF = 0, BOUNCE_PRIMARY = 1, BOUNCE_SECONDARY = 2;  // TraceParams::bounce_mode
constexpr int TILE_W = 8, TILE_H = 4;
constexpr int WARPS_PER_BLOCK = 4;
constexpr int N_BINS = 8;            // chord-length classes of the ray list (longest first)
constexpr uint32_t HIT_CHUNK = 8;   // hit slots a lane takes from the stream at a time (one atomic per chunk)
constexpr uint32_t HIT_NONE = 0xffffffffu;
// Resident marching blocks per SM the register budget is sized for (65536 registers / (128 threads x 5) = 96 registers).
// The Volumetric kernels fit without spills since their state touched only at surfaces, level switches and refills
// moved to shared memory.  With that state in registers they spilled a few dozen bytes; 4 blocks (no spills) were then
// measured on an H100 SXM (700 W) 2.5 % faster on the C2 bench frame but 3-4 % slower on C1 and C3, so 5 stays.
constexpr int MIN_BLOCKS_PER_SM = 5;
// The marching loop's exits (TraceParams::event_threshold, tail_divisor, refill_threshold; launch_trace sets them):
// leave the loop once 24 lanes wait; once the ray list is exhausted, once half of the lanes that still have a ray
// wait; and run the lean per-lane loop once at most 4 lanes of a warp still march.
constexpr uint32_t EVENT_THRESHOLD = 24, TAIL_DIVISOR = 2, REFILL_THRESHOLD = 4;


constexpr double D_INF = __builtin_huge_val();

// Programmatic dependent launch: the frame's kernels are launched back to back with
// cudaLaunchAttributeProgrammaticStreamSerialization, so a kernel's blocks may become resident while the previous
// kernel is still draining; every kernel lets its successor in at once and waits here — until the previous grid has
// completed and its writes are visible — before it touches anything that grid produced.  Without the attribute both
// instructions do nothing.
__device__ __forceinline__ void grid_dependency_sync() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

struct Ray {
    double ox, oy, oz, dx, dy, dz;   // original ray
    double tdx, tdy, tdz;            // t_delta = 1/|d| (raycast.rs:769)
    double half_over_len;            // 0.5 / |d| (raycast.rs:669)
    int sx, sy, sz;                  // signum_101(d) (raycast.rs:768)
};

// State::* of the active raycaster (raycast.rs:99-121); the cube is kept relative to the lower
// corner of its level so that the bounds test is one unsigned compare.
struct Caster {
    double tmx, tmy, tmz;
    double last_t;
    int rx, ry, rz;
    int face;        // Face7 through which the current cube was entered
    uint32_t idx;    // linear index of the current cube in its volume (+ brick offset on the inner level)
};

// Geometry of one level as the DDA needs it.
struct Level {
    int lox, loy, loz;
    int nx, ny, nz;    // sizes
    uint32_t base;
};

AICB_DEV uint4 ld_stream(const uint4 *p) { return __ldg(p); }
AICB_DEV void st_stream(uint4 *p, uint4 v) { *p = v; }

AICB_DEV int signum_101(double x) { return (x == 0.0 || x != x) ? 0 : (x < 0.0 ? -1 : 1); }

// a / b, correctly rounded, given rb = RN(1 / b): two Newton corrections with exact remainders (Markstein: with a
// correctly rounded reciprocal and a faithful quotient, q + (a - b q) rb rounds to RN(a / b)).  The ray's t_delta IS
// RN(1 / |direction|) (raycast.rs:769), so the divisions by the direction in Raycaster::within / fast_forward /
// scale_to_integer_step cost five FP64 instructions instead of a division routine.  Outside a generous exponent
// window (where an intermediate could leave the normal range) the real division is used.  The window bounds |a| from
// below as well: with 2^-600 <= |a| the quotient is at least 2^-1001 and the remainders are multiples of 2^-705, so
// all stay normal and exact; a quotient near the subnormal range would not be correctly rounded.  Zeros take the
// division too (the corrections would turn -0 / b into +0).  Of the callers, pixel_ray's numerators are integers
// (0 among them) and scale_to_integer_step's are >= 2^-53; caster_begin's and project_ndc's can be zero, and can be
// tiny only for a ray origin within 2^-600 of a grid plane or a degenerate camera matrix.
// tests/test_gpu_scalar_math.py checks it against IEEE division on every pixel quotient x / W with W <= 16384, on
// random pairs with |b| from 2^-420 to 2^420 and |a| from 2^-1074 to 2^210, and on project_ndc's three quotients.
AICB_DEV double div_known_recip(double a, double b, double rb) {
    const double ab = fabs(b), aa = fabs(a);
    if (!((ab >= 0x1p-400) & (ab <= 0x1p400) & (aa <= 0x1p200) & (aa >= 0x1p-600))) return a / b;
    const double q0 = a * rb;
    const double r0 = fma(-b, q0, a);
    const double q1 = fma(r0, rb, q0);
    const double r1 = fma(-b, q1, a);
    return fma(r1, rb, q1);
}

// scale_to_integer_step (raycast.rs:797-819). fmod(s, 1) == s - trunc(s) exactly.  rds = RN(1 / |ds|).
AICB_DEV double scale_to_integer_step(double s, double ds, double rds) {
    if (ds == 0.0 && !(s != s)) return D_INF;
    if (ds < 0.0) {
        s = -s;
        ds = -ds;
    }
    double r = s - trunc(s);
    if (r < 0.0) r = r + 1.0;
    return div_known_recip(1.0 - r, ds, rds);
}

// 1 / res for res = 2^k (Resolution::recip_f64): exact, no division
AICB_DEV double recip_pow2(int res) { return __hiloint2double((1023 - (31 - __clz(res))) << 20, 0); }

AICB_DEV bool in_i32_range(double x) { return (-2147483648.0 <= x) & (x < 2147483648.0); }
AICB_DEV double rclamp01(double v) { return v < 0.0 ? 0.0 : (v > 1.0 ? 1.0 : v); }  // NaN passes through

AICB_DEV float ps_mul(float a, float b) {
    float v = a * b;
    return (v != v) ? 0.0f : v;
}
AICB_DEV float ps_clamped(float v) { return (v > 0.0f) ? v : 0.0f; }
AICB_DEV float zo_clamped(float v) {
    if (v > 0.0f && v <= 1.0f) return v;
    if (v <= 0.0f) return 0.0f;
    return 1.0f;
}

AICB_DEV bool tmax_valid(const Caster &c, const Ray &r) {  // valid_for_stepping (raycast.rs:563-570)
    const bool any_nan = (c.tmx != c.tmx) | (c.tmy != c.tmy) | (c.tmz != c.tmz);
    const bool any_fin = isfinite(c.tmx) | isfinite(c.tmy) | isfinite(c.tmz);
    return ((r.sx | r.sy | r.sz) != 0) & !any_nan & any_fin;
}

// Raycaster::new(...).within(bounds, true) (raycast.rs:196-230, 513-545, 632-704) followed by the
// FirstLast::Beginning part of next() (raycast.rs:255-263): advance until the first in-bounds
// cube.  Returns false when the iterator produces nothing.  *valid = valid_for_stepping().
// Inlined: as a call, its Ray and Caster went through a 160-byte stack frame per thread (100 KB of local memory per SM
// in trace_kernel, competing with the cell, brick and ray loads for L1) and every field was a local load or store.
AICB_DEV bool caster_begin(Caster &c, const Ray &r, double ox, double oy, double oz, const Level lv, bool *valid) {
    *valid = false;
    if (!(in_i32_range(ox) & in_i32_range(oy) & in_i32_range(oz))) return false;  // Cube::containing -> EMPTY
    {
        int fx = __double2int_rd(ox), fy = __double2int_rd(oy), fz = __double2int_rd(oz);
        const int lo = INT32_MIN + 1, hi = INT32_MAX - 1;
        if ((fx < lo) | (fx >= hi) | (fy < lo) | (fy >= hi) | (fz < lo) | (fz >= hi)) return false;  // MAXIMUM_BOUNDS filter
    }
    if (lv.nx <= 0 || lv.ny <= 0 || lv.nz <= 0) return false;  // ORIGIN_EMPTY

    // fast_forward: (plane - origin) / direction per moving axis; the dot products with an axis
    // normal reduce exactly to this quotient.
    double max_t = 0.0;
    if (r.sx != 0) max_t = fmax(max_t, div_known_recip((double)(r.sx < 0 ? lv.lox + lv.nx : lv.lox) - ox, r.dx, r.sx < 0 ? -r.tdx : r.tdx));
    if (r.sy != 0) max_t = fmax(max_t, div_known_recip((double)(r.sy < 0 ? lv.loy + lv.ny : lv.loy) - oy, r.dy, r.sy < 0 ? -r.tdy : r.tdy));
    if (r.sz != 0) max_t = fmax(max_t, div_known_recip((double)(r.sz < 0 ? lv.loz + lv.nz : lv.loz) - oz, r.dz, r.sz < 0 ? -r.tdz : r.tdz));

    double px = ox, py = oy, pz = oz, t0 = 0.0;
    if (max_t > 0.0) {
        double t_start = max_t - r.half_over_len;
        if (!isfinite(t_start)) t_start = max_t;
        px = ox + r.dx * t_start;  // Ray::advance (ray.rs:107-112)
        py = oy + r.dy * t_start;
        pz = oz + r.dz * t_start;
        if (!(in_i32_range(px) & in_i32_range(py) & in_i32_range(pz))) return false;
        t0 = t_start;
    }
    int cx = __double2int_rd(px), cy = __double2int_rd(py), cz = __double2int_rd(pz);
    c.tmx = scale_to_integer_step(px, r.dx, r.tdx) + t0;
    c.tmy = scale_to_integer_step(py, r.dy, r.tdy) + t0;
    c.tmz = scale_to_integer_step(pz, r.dz, r.tdz) + t0;
    c.last_t = t0;
    c.face = AICB_FACE_WITHIN;
    const bool ok = tmax_valid(c, r);
    *valid = ok;

    const int hx = lv.lox + lv.nx, hy = lv.loy + lv.ny, hz = lv.loz + lv.nz;
    for (;;) {
        // is_out_of_bounds_ahead (raycast.rs:711-728)
        bool xl = cx < lv.lox, xh = cx >= hx;
        bool yl = cy < lv.loy, yh = cy >= hy;
        bool zl = cz < lv.loz, zh = cz >= hz;
        bool enter = (r.sx == 0 ? (xl | xh) : (r.sx < 0 ? xh : xl)) | (r.sy == 0 ? (yl | yh) : (r.sy < 0 ? yh : yl)) |
                     (r.sz == 0 ? (zl | zh) : (r.sz < 0 ? zh : zl));
        bool exit_ = (r.sx == 0 ? (xl | xh) : (r.sx < 0 ? xl : xh)) | (r.sy == 0 ? (yl | yh) : (r.sy < 0 ? yl : yh)) |
                     (r.sz == 0 ? (zl | zh) : (r.sz < 0 ? zl : zh));
        if (exit_) return false;
        if (!enter) break;
        if (!ok) return false;
        // State::step (raycast.rs:577-626)
        if (c.tmx < c.tmy) {
            if (c.tmx < c.tmz) { c.last_t = c.tmx; cx += r.sx; c.tmx += r.tdx; c.face = r.sx > 0 ? AICB_FACE_NX : AICB_FACE_PX; }
            else               { c.last_t = c.tmz; cz += r.sz; c.tmz += r.tdz; c.face = r.sz > 0 ? AICB_FACE_NZ : AICB_FACE_PZ; }
        } else {
            if (c.tmy < c.tmz) { c.last_t = c.tmy; cy += r.sy; c.tmy += r.tdy; c.face = r.sy > 0 ? AICB_FACE_NY : AICB_FACE_PY; }
            else               { c.last_t = c.tmz; cz += r.sz; c.tmz += r.tdz; c.face = r.sz > 0 ? AICB_FACE_NZ : AICB_FACE_PZ; }
        }
    }
    c.rx = cx - lv.lox;
    c.ry = cy - lv.loy;
    c.rz = cz - lv.loz;
    c.idx = lv.base + (uint32_t)((c.rx * lv.ny + c.ry) * lv.nz + c.rz);
    return true;
}

// One State::step (raycast.rs:577-626) on the active caster, with incremental index update; select-based so that
// lanes stepping along different axes stay converged.  Axis choice as the reference: x if t_max.x is strictly the
// smallest, else y if t_max.y < t_max.z, else z.
// Returns true if the new cube is outside the level (the "exit" step of raycast.rs:265-274).
AICB_DEV bool caster_step(Caster &c, const Ray &r, int nx, int ny, int nz) {
    const bool xy = c.tmx < c.tmy, xz = c.tmx < c.tmz, yz = c.tmy < c.tmz;
    const bool ax = xy & xz;
    const bool ay = !xy & yz;
    const bool az = !(ax | ay);
    const double tm = ax ? c.tmx : (ay ? c.tmy : c.tmz);
    const double td = ax ? r.tdx : (ay ? r.tdy : r.tdz);
    const double nt = tm + td;
    c.last_t = tm;
    c.tmx = ax ? nt : c.tmx;
    c.tmy = ay ? nt : c.tmy;
    c.tmz = az ? nt : c.tmz;
    const int sg = ax ? r.sx : (ay ? r.sy : r.sz);
    c.rx += ax ? sg : 0;
    c.ry += ay ? sg : 0;
    c.rz += az ? sg : 0;
    const int stride = ax ? ny * nz : (ay ? nz : 1);
    c.idx += (uint32_t)(sg * stride);
    c.face = (ax ? AICB_FACE_NX : (ay ? AICB_FACE_NY : AICB_FACE_NZ)) + (sg > 0 ? 0 : 3);
    const int pos = ax ? c.rx : (ay ? c.ry : c.rz);
    const int lim = ax ? nx : (ay ? ny : nz);
    return (uint32_t)pos >= (uint32_t)lim;
}

// ---- light ---------------------------------------------------------------------------------------
constexpr uint32_t TEXEL_ONE = 144u | (144u << 8) | (144u << 16) | (255u << 24);       // PackedLight::ONE
constexpr uint32_t TEXEL_NO_RAYS = (1u << 24);
constexpr uint32_t TEXEL_UNINIT = 0u;

// BlockSky::light_outside (sky.rs:113-147)
AICB_DEV uint32_t light_outside(const DeviceScene &s, int x, int y, int z) {
    const int c[3] = {x, y, z};
    int n_equal = 0, n_less = 0, which = 0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        int beyond = s.lo[a] - 1;
        int hi = s.lo[a] + s.size[a];
        if (beyond == c[a]) { n_equal++; which = a; } else if (beyond < c[a]) n_less++;
        if (c[a] == hi) { n_equal++; which = 3 + a; } else if (c[a] < hi) n_less++;
    }
    if (n_less == 6) return TEXEL_UNINIT;
    if (n_equal == 1 && n_less == 5) return s.sky_faces[which];
    return TEXEL_NO_RAYS;
}

// SpaceRaytracer::get_packed_light (sr.rs:241-246)
AICB_NOINLINE uint32_t get_packed_light(const DeviceScene &s, int x, int y, int z, uint32_t &texels) {
    uint32_t dx = (uint32_t)(x - s.lo[0]), dy = (uint32_t)(y - s.lo[1]), dz = (uint32_t)(z - s.lo[2]);
    if ((dx >= (uint32_t)s.size[0]) | (dy >= (uint32_t)s.size[1]) | (dz >= (uint32_t)s.size[2]))
        return light_outside(s, x, y, z);
    if (s.light == nullptr) return TEXEL_ONE;
    texels++;
    return __ldg(s.light + ((size_t)dx * s.size[1] + dy) * s.size[2] + dz);
}

AICB_DEV void texel_value_ao(const float *lut, uint32_t t, float out[4]) {  // data.rs:145-158
    out[0] = lut[t & 255];
    out[1] = lut[(t >> 8) & 255];
    out[2] = lut[(t >> 16) & 255];
    uint32_t st = t >> 24;
    out[3] = (st == 255) ? 1.0f : (st == 128 ? 0.25f : 0.0f);
}

// f64::rem_euclid(1.0): r = x % 1.0 (fmod: exact, with x's sign, so -0 for a negative integer or -0), + 1 if r < 0.
// x - trunc(x) is that remainder exactly except for its zeros, which it makes +0; copysign restores fmod's -0.
// tests/test_gpu_scalar_math.py checks it against fmod around the integers, 2^52 .. 2^53 and beyond, both signs.
AICB_DEV double rem_euclid1(double x) {
    const double r = copysign(x - trunc(x), x);
    return r < 0.0 ? r + 1.0 : r;
}

// get_interpolated_light (sr.rs:248-359). `lut` is the shared-memory copy of the decode table.
// Written for the convergent shading kernel: no dynamically indexed arrays, and the (up to) eight texel loads of
// the two layers are issued together before any of them is used.
AICB_DEV void interpolated_light(const DeviceScene &s, const float *lut, uint32_t mode, int cube_x, int cube_y,
                                 int cube_z, int face, double spx, double spy, double spz, float out[3],
                                 uint32_t *texels_out) {
    const double eps = 0.5 / 256.0;
    const double sp[3] = {spx, spy, spz};
    // Face::rotation_from_nz (face.rs:395-405): axis + sign of the images of +X and +Y, and the normal
    //   NX: RYZX   NY: RZXY   NZ: RXYZ   PX: RyZx   PY: RZxy   PZ: RXyz   Within: IDENTITY, normal 0
    const bool within = face == AICB_FACE_WITHIN;
    const int fa = within ? 2 : (face - 1) % 3;            // axis of the normal
    const int a1 = fa == 0 ? 1 : (fa == 1 ? 2 : 0);
    const int a2 = fa == 0 ? 2 : (fa == 1 ? 0 : 1);
    const int an = fa;
    const int sn = within ? 0 : (face >= AICB_FACE_PX ? 1 : -1);
    int s1 = (face == AICB_FACE_PX) ? -1 : 1;
    int s2 = (face == AICB_FACE_PY || face == AICB_FACE_PZ) ? -1 : 1;
    const double sp1 = a1 == 0 ? sp[0] : (a1 == 1 ? sp[1] : sp[2]);
    const double sp2 = a2 == 0 ? sp[0] : (a2 == 1 ? sp[1] : sp[2]);
    const double spn = an == 0 ? sp[0] : (an == 1 ? sp[1] : sp[2]);
    double mix_1 = rem_euclid1((s1 > 0 ? sp1 : -sp1) - 0.5);
    double mix_2 = rem_euclid1((s2 > 0 ? sp2 : -sp2) - 0.5);
    if (mix_1 > 0.5) { mix_1 = 1.0 - mix_1; s1 = -s1; }
    if (mix_2 > 0.5) { mix_2 = 1.0 - mix_2; s2 = -s2; }
    if (mode == AICB_LIGHT_COARSE) {          // surface.rs:510-514
        double f1 = floor(mix_1 * 4.0), f2 = floor(mix_2 * 4.0);
        f1 = f1 < 0.0 ? 0.0 : (f1 > 3.0 ? 3.0 : f1);
        f2 = f2 < 0.0 ? 0.0 : (f2 > 3.0 ? 3.0 : f2);
        mix_1 = (f1 + 0.5) / 4.0;
        mix_2 = (f2 + 0.5) / 4.0;
    } else if (mode == AICB_LIGHT_SMOOTHSTEP) {  // surface.rs:517-520
        double c1 = rclamp01(mix_1), c2 = rclamp01(mix_2);
        mix_1 = 3.0 * (c1 * c1) - 2.0 * ((c1 * c1) * c1);
        mix_2 = 3.0 * (c2 * c2) - 2.0 * ((c2 * c2) * c2);
    }
    const float m1 = (float)mix_1, m2 = (float)mix_2;

    const int cube_n = an == 0 ? cube_x : (an == 1 ? cube_y : cube_z);
    const double fdot_sp = sn == 0 ? 0.0 : (sn > 0 ? spn : -spn);
    const double ctr = (double)cube_n + 0.5;
    const double fdot_c = sn == 0 ? 0.0 : (sn > 0 ? ctr : -ctr);
    const double height_in_cube = fdot_sp - fdot_c + 0.5;
    const bool two_layers = !(height_in_cube > (1.0 - eps));

    // the two candidate coordinates along each role: [0] = lo / front layer, [1] = hi / back layer
    const double q1[2] = {sp1 + (double)s1 * -0.5, sp1 + (double)s1 * 0.5};
    const double q2[2] = {sp2 + (double)s2 * -0.5, sp2 + (double)s2 * 0.5};
    const double qn[2] = {sn != 0 ? spn + (double)sn * (1.0 - eps) : spn, sn != 0 ? spn + (double)sn * eps : spn};
    bool ok1[2], ok2[2], okn[2];
    int i1[2], i2[2], in_[2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
        ok1[j] = in_i32_range(q1[j]); i1[j] = __double2int_rd(q1[j]);
        ok2[j] = in_i32_range(q2[j]); i2[j] = __double2int_rd(q2[j]);
        okn[j] = in_i32_range(qn[j]); in_[j] = __double2int_rd(qn[j]);
    }
    // issue the loads: tex[layer][k], k: 0 near12, 1 near1far2, 2 near2far1, 3 far12
    uint32_t tex[2][4];
    uint32_t texels = 0;
#pragma unroll
    for (int layer = 0; layer < 2; layer++) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int j1 = (k >> 1) & 1, j2 = k & 1;
            const int c1 = i1[j1], c2 = i2[j2], cn = in_[layer];
            const int x = a1 == 0 ? c1 : (a2 == 0 ? c2 : cn);
            const int y = a1 == 1 ? c1 : (a2 == 1 ? c2 : cn);
            const int z = a1 == 2 ? c1 : (a2 == 2 ? c2 : cn);
            uint32_t t = s.sky_mean;
            if ((layer == 0 || two_layers) && (ok1[j1] & ok2[j2] & okn[layer])) {
                const uint32_t dx = (uint32_t)(x - s.lo[0]), dy = (uint32_t)(y - s.lo[1]), dz = (uint32_t)(z - s.lo[2]);
                if ((dx >= (uint32_t)s.size[0]) | (dy >= (uint32_t)s.size[1]) | (dz >= (uint32_t)s.size[2])) {
                    t = light_outside(s, x, y, z);
                } else if (s.light == nullptr) {
                    t = TEXEL_ONE;
                } else {
                    texels++;
                    t = __ldg(s.light + ((size_t)dx * s.size[1] + dy) * s.size[2] + dz);
                }
            }
            tex[layer][k] = t;
        }
    }
    float front[4], result[4];
#pragma unroll
    for (int layer = 0; layer < 2; layer++) {
        if (layer == 1 && !two_layers) break;
        uint32_t t3 = tex[layer][3];
        if ((tex[layer][1] >> 24) != 255 && (tex[layer][2] >> 24) != 255) t3 = tex[layer][0];  // sr.rs:317-321
        float v0[4], v1[4], v2[4], v3[4], cur[4];
        texel_value_ao(lut, tex[layer][0], v0);
        texel_value_ao(lut, tex[layer][1], v1);
        texel_value_ao(lut, tex[layer][2], v2);
        texel_value_ao(lut, t3, v3);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            float ab = v0[i] + (v1[i] - v0[i]) * m2;
            float cd = v2[i] + (v3[i] - v2[i]) * m2;
            cur[i] = ab + (cd - ab) * m1;
        }
        if (layer == 0) {
#pragma unroll
            for (int i = 0; i < 4; i++) { front[i] = cur[i]; result[i] = cur[i]; }
        } else {
            const float h = (float)height_in_cube;
#pragma unroll
            for (int i = 0; i < 4; i++) result[i] = cur[i] + (front[i] - cur[i]) * h;
        }
    }
    const float w = fmaxf(result[3], 0.1f);
#pragma unroll
    for (int i = 0; i < 3; i++) {
        float v = result[i] / w;
        out[i] = (v == 0.0f) ? 0.0f : v;
    }
    *texels_out = texels;
}

// Rgba::from(ColorBuf) (raytracer_components.rs:122-146)
AICB_DEV void colorbuf_to_rgba(float l0, float l1, float l2, float tr, float out[4]) {
    if (tr >= 1.0f) { out[0] = out[1] = out[2] = out[3] = 0.0f; return; }
    float alpha = 1.0f - tr;
    float c[3] = {l0 / alpha, l1 / alpha, l2 / alpha};
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        if (c[i] > 0.0f) {} else if (c[i] == 0.0f) c[i] = 0.0f; else ok = false;
    }
    if (!ok) { c[0] = 1.0f; c[1] = 0.0f; c[2] = 0.0f; }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2];
    out[3] = (alpha > 0.0f && alpha <= 1.0f) ? alpha : (alpha == 0.0f ? 0.0f : 1.0f);
}

// Two f16 texel channels as one word, lo in the low half: half::f16::from_f32 of each (round to nearest even, overflow
// to infinity, subnormals kept).  tests/test_gpu_scalar_math.py checks it on every f32 bit pattern.
AICB_DEV uint32_t f16x2_texel(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&h);
}

AICB_DEV unsigned char sat_u8(float v) {  // `as u8`: saturating, NaN -> 0
    if (!(v > 0.0f)) return 0;
    if (v >= 255.0f) return 255;
    return (unsigned char)v;
}

// component_to_srgb8 (color.rs:1038-1054) as a search: thr[k] (k = 1..255) is the smallest f32 whose
// encoding is >= k, computed on the host with the platform powf; the encoding is monotone in c.
AICB_DEV unsigned char component_to_srgb8(const float *thr, float c) {
    int lo = 0, hi = 255;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int mid = (lo + hi + 1) >> 1;
        if (c >= thr[mid]) lo = mid; else hi = mid - 1;
    }
    return (unsigned char)lo;
}

// Camera::post_process_color (camera_struct.rs:376-382, graphics_options.rs:352-368) of rgba's colour; alpha is kept
AICB_DEV void post_process_color(const TraceParams &P, const float rgba[4], float c[3]) {
    c[0] = ps_mul(rgba[0], P.exposure); c[1] = ps_mul(rgba[1], P.exposure); c[2] = ps_mul(rgba[2], P.exposure);
    if (isfinite(P.maximum_intensity)) {
        if (P.tone_mapping == AICB_TONE_CLAMP) {
#pragma unroll
            for (int i = 0; i < 3; i++) c[i] = c[i] > P.maximum_intensity ? P.maximum_intensity : c[i];
        } else {
            float lum = c[1] * 0.7152f + (c[0] * 0.2126f + c[2] * 0.0722f);
            float s = ps_clamped(1.0f / (1.0f + lum / P.maximum_intensity));
#pragma unroll
            for (int i = 0; i < 3; i++) c[i] = ps_mul(c[i], s);
        }
    }
}

// Camera::post_process_color + to_srgb8 (camera_struct.rs:376-382, color.rs:669-676)
AICB_DEV uchar4 encode_srgb8(const TraceParams &P, const float *thr, float l0, float l1, float l2, float tr) {
    float rgba[4];
    colorbuf_to_rgba(l0, l1, l2, tr, rgba);
    float c[3];
    post_process_color(P, rgba, c);
    return make_uchar4(component_to_srgb8(thr, c[0]), component_to_srgb8(thr, c[1]), component_to_srgb8(thr, c[2]),
                       sat_u8(roundf(rgba[3] * 255.0f)));
}

// Camera::project_ndc_into_world (camera_struct.rs:238-257); euclid transform_point3d
AICB_DEV void project_ndc(const TraceParams &P, double x, double y, double z, double out[3]) {
    const double *m = P.m;
    double hx = x * m[0] + y * m[4] + z * m[8] + m[12];
    double hy = x * m[1] + y * m[5] + z * m[9] + m[13];
    double hz = x * m[2] + y * m[6] + z * m[10] + m[14];
    double hw = x * m[3] + y * m[7] + z * m[11] + m[15];
    if (hw > 0.0) {   // three quotients by the same w: one division for RN(1 / w), then exact quotients from it
        const double rw = 1.0 / hw;
        out[0] = div_known_recip(hx, hw, rw); out[1] = div_known_recip(hy, hw, rw); out[2] = div_known_recip(hz, hw, rw);
    } else {
        out[0] = out[1] = out[2] = __longlong_as_double(0x7ff8000000000000LL);
    }
}

// viewport.rs:104-113 + renderer.rs:424-451,489-491.  The four quotients by the framebuffer size are correctly rounded
// from the host's RN(1 / W) and RN(1 / H) (pixel coordinates and sizes are integers < 2^32, well inside
// div_known_recip's exponent window, or 0, which it divides), so they equal the divisions bit for bit.
AICB_DEV void pixel_ray(const TraceParams &P, uint32_t xch, uint32_t ych, int sample, double o[3], double d[3]) {
    const double W = (double)P.fb_width, H = (double)P.fb_height;
    const double x0 = div_known_recip((double)xch, W, P.inv_width) * 2.0 - 1.0;
    const double x1 = div_known_recip((double)(xch + 1), W, P.inv_width) * 2.0 - 1.0;
    const double y0 = -(div_known_recip((double)ych, H, P.inv_height) * 2.0 - 1.0);
    const double y1 = -(div_known_recip((double)(ych + 1), H, P.inv_height) * 2.0 - 1.0);
    double px, py;
    if (sample < 0) {
        px = (x0 + x1) / 2.0;
        py = (y0 + y1) / 2.0;
    } else {
        const double u = (sample == 0) ? 1. / 8. : (sample == 1) ? 3. / 8. : (sample == 2) ? 5. / 8. : 7. / 8.;
        const double v = (sample == 0) ? 5. / 8. : (sample == 1) ? 1. / 8. : (sample == 2) ? 7. / 8. : 3. / 8.;
        px = x0 + (x1 - x0) * u;
        py = y0 + (y1 - y0) * v;
    }
    double nearp[3], farp[3];
    project_ndc(P, px, py, 0.0, nearp);
    project_ndc(P, px, py, 1.0, farp);
    o[0] = nearp[0]; o[1] = nearp[1]; o[2] = nearp[2];
    d[0] = farp[0] - nearp[0]; d[1] = farp[1] - nearp[1]; d[2] = farp[2] - nearp[2];
}

// Conservative, division-free test that a ray cannot touch the Space: the slab test against the bounds grown by 1/64
// cube, with the entry / exit parameters compared by cross-multiplication.  True only when the exact-arithmetic ray
// misses the grown box (f64 rounding of the products is ~1e-13 relative, the margin ~1e-2 absolute), in which case
// Raycaster::within (raycast.rs:632-704) cannot produce a cube either: its positions are accurate to far less than the
// margin.  Any NaN / infinity makes every comparison false and the ray takes the exact path.  Two thirds of the rays of
// the bench frame never enter the Space; for them this replaces 10 divisions, 2 square roots and Raycaster::within.
AICB_DEV bool certainly_misses(const double o[3], const double d[3], const DeviceScene &S) {
    const double M = 1.0 / 64.0;
    double n_in[3], n_out[3], ad[3];
    bool moving[3];
    bool miss = false;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double lo = (double)S.lo[a] - M, hi = (double)S.lo[a] + (double)S.size[a] + M;
        ad[a] = fabs(d[a]);
        moving[a] = ad[a] > 0.0;
        n_in[a] = d[a] > 0.0 ? lo - o[a] : o[a] - hi;     // t_in  = n_in  / |d|
        n_out[a] = d[a] > 0.0 ? hi - o[a] : o[a] - lo;    // t_out = n_out / |d|
        if (!moving[a]) miss |= (o[a] < lo) | (o[a] > hi);
        else miss |= n_out[a] < 0.0;                       // the grown box lies behind the origin
    }
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b = 0; b < 3; b++) {
            if (a == b) continue;
            // t_in[a] > t_out[b]  <=>  n_in[a] |d_b| > n_out[b] |d_a|   (both |d| > 0)
            const double l = n_in[a] * ad[b], r = n_out[b] * ad[a];
            if (moving[a] & moving[b]) miss |= l > r + 1e-9 * (fabs(l) + fabs(r));
        }
    return miss;
}

// ---- per-lane state ----------------------------------------------------------------------------------
template <bool AUX>
struct AuxState {};
template <>
struct AuxState<true> {
    uint32_t n_outer, n_inner, n_blocks;   // device counters of the roofline accounting
};

// A lane is marching, parked (waiting for the warp to serve its level switch / to take its result), or has no ray.
enum LaneState : int { ST_IDLE = 0, ST_MARCH = 1, ST_ENTER = 2, ST_POP = 3, ST_DONE = 4, ST_EXHAUSTED = 5 };

// task -> pixel mapping shared by the three kernels: pixel tasks are tile-ordered (32 consecutive
// pixel tasks = one 8x4 tile); returns false for the padding pixels of edge tiles.  With a pixel list (LIST
// instantiations only, so that the kernels of other frames do not carry the branch) pixel task i is the listed pixel
// and its outputs go to position i; a warp then takes 32 consecutive list entries.
template <bool LIST>
AICB_DEV bool task_pixel(const TraceParams &P, uint32_t pixel_task, uint32_t *px, uint32_t *py, size_t *out_index) {
    if (P.rays) {
        *px = *py = 0;
        *out_index = pixel_task;
        return pixel_task < P.n_rays;
    }
    if (LIST && P.target.pixel_list) {
        if (pixel_task >= P.target.n_list) return false;
        const uint32_t v = __ldg(P.target.pixel_list + pixel_task);
        *px = v % P.fb_width;
        *py = v / P.fb_width;
        *out_index = pixel_task;
        return true;
    }
    const uint32_t tile = pixel_task >> 5, in_tile = pixel_task & 31;
    const uint32_t tx = tile % P.tiles_x, ty = tile / P.tiles_x;
    const uint32_t x = tx * TILE_W + (in_tile & (TILE_W - 1));
    const uint32_t ly = ty * TILE_H + (in_tile / TILE_W);
    uint32_t y = ly;
    if (P.shard_count > 1) {  // local row -> framebuffer row (row-strip sharding)
        const uint32_t strip_local = ly / P.strip_rows;
        y = (strip_local * P.shard_count + P.shard_index) * P.strip_rows + ly % P.strip_rows;
    }
    *px = x;
    *py = y;
    *out_index = P.out_full_frame ? (size_t)y * P.fb_width + x : (size_t)ly * P.fb_width + x;
    return x < P.fb_width && ly < P.local_rows;
}

// ======================================================================================================
// Kernel 1 — ray generation: pixel -> NDC patch -> world ray (viewport.rs:104-113, renderer.rs:424-451,
// camera_struct.rs:238-257), trace_ray_impl's prologue (sr.rs:135-180) and the outer
// Raycaster::new().within(space bounds) (raycast.rs:196-230, 632-704).  One thread per ray, fully convergent.
// ======================================================================================================
static __global__ void __launch_bounds__(128) gen_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    grid_dependency_sync();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = i < n_chunk_tasks;
    const uint32_t task = P.task_base + i;
    const uint32_t pixel_task = task / P.n_samples, sample = task % P.n_samples;
    RayRecordA rec;
    RayRecordB rb;
    uint32_t px, py;
    size_t out_index;
    bool active = in_range && task_pixel<true>(P, pixel_task, &px, &py, &out_index);
    if (P.bounce_mode == BOUNCE_SECONDARY && active) active = P.bounce_req[i] != HIT_NONE;   // no surface to light
    rec.flags = 0;
    bool running = false;
    uint32_t octant = 0;
    int bin = 0;
    if (active) {
        const DeviceScene &S = P.scene;
        double o[3], d[3];
        if (P.rays) {
            const double *rp = P.rays + 6 * (size_t)pixel_task;
            o[0] = rp[0]; o[1] = rp[1]; o[2] = rp[2]; d[0] = rp[3]; d[1] = rp[4]; d[2] = rp[5];
        } else {
            pixel_ray(P, px, py, P.n_samples == 4 ? (int)sample : -1, o, d);
        }
        // Sky::sample octant (sky.rs:32-41) and the t conversions (sr.rs:146-151) use the original direction
        octant = ((d[0] >= 0.0) << 2) + ((d[1] >= 0.0) << 1) + (d[2] >= 0.0);
        const double d_orig[3] = {d[0], d[1], d[2]};
        // Parameters::new (raycast.rs:749-771)
        if (!((fabs(d[0]) < 1e100) & (fabs(d[1]) < 1e100) & (fabs(d[2]) < 1e100))) { d[0] = d[1] = d[2] = 0.0; }
    if (!certainly_misses(o, d, S)) {
        rec.t_to_abs = sqrt(d_orig[0] * d_orig[0] + d_orig[1] * d_orig[1] + d_orig[2] * d_orig[2]);
        rec.t_to_view = (float)(rec.t_to_abs / P.view_distance);
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
        Caster c;
        c.tmx = c.tmy = c.tmz = c.last_t = 0.0;
        c.rx = c.ry = c.rz = 0;
        c.face = 0;
        c.idx = 0;
        bool valid;
        running = caster_begin(c, r, o[0], o[1], o[2], lv, &valid);
        rec.ox = r.ox; rec.oy = r.oy; rec.oz = r.oz; rec.dx = r.dx; rec.dy = r.dy; rec.dz = r.dz;
        rb.tdx = r.tdx; rb.tdy = r.tdy; rb.tdz = r.tdz;
        rb.half_over_len = r.half_over_len;
        rb.tmx = c.tmx; rb.tmy = c.tmy; rb.tmz = c.tmz; rb.last_t = c.last_t;
        rb.rx = c.rx; rb.ry = c.ry; rb.rz = c.rz;
        rb.task = i;
        rec.flags = ((uint32_t)c.face & 7u) | (running ? 8u : 0u) | (valid ? 16u : 0u) | 32u | ((uint32_t)(r.sx + 1) << 6) |
                    ((uint32_t)(r.sy + 1) << 8) | ((uint32_t)(r.sz + 1) << 10) | (octant << 12);
        if (running) {
            // Scheduling heuristic only (never affects results): the number of cube boundaries the ray's chord
            // through the space bounds crosses, in f32.  Long rays are listed in early bins so that the marching
            // kernel starts them first and the frame does not end on a few long serial chains.
            const float lo3[3] = {(float)lv.lox, (float)lv.loy, (float)lv.loz};
            const float n3[3] = {(float)lv.nx, (float)lv.ny, (float)lv.nz};
            float tn = 0.0f, tf = 3.0e38f, l1 = 0.0f;
#pragma unroll
            for (int a = 0; a < 3; a++) {
                const float da = (float)d[a], oa = (float)o[a];
                if (da != 0.0f) {
                    const float t0 = (lo3[a] - oa) / da, t1 = (lo3[a] + n3[a] - oa) / da;
                    tn = fmaxf(tn, fminf(t0, t1));
                    tf = fminf(tf, fmaxf(t0, t1));
                    l1 += fabsf(da);
                }
            }
            const float crossings = fmaxf(tf - tn, 0.0f) * l1;
            const float frac = crossings / (n3[0] + n3[1] + n3[2]);
            int q = (int)(frac * (float)N_BINS);
            q = q < 0 ? 0 : (q > N_BINS - 1 ? N_BINS - 1 : q);
            bin = N_BINS - 1 - q;
        }
    }   // (!certainly_misses)
    }
    // Rays that enter the space go to the marching kernel through the binned list (warp-aggregated append); all
    // others are complete already: nothing hit, transmittance 1, no steps.  The listed rays of a warp take
    // consecutive record indices, so that their records are whole lines (a record at the task index would leave the
    // ~1/3 of the lanes that write spread over 32 records, every line and sector written in pieces).
    const unsigned listed = __ballot_sync(0xffffffffu, running);
    if (running) {
        const int lane = (int)(threadIdx.x & 31);
        const unsigned below = listed & ((1u << lane) - 1u);
        uint32_t rbase = 0;
        if (below == 0) rbase = atomicAdd(P.ray_counter, (unsigned)__popc(listed));
        rbase = __shfl_sync(listed, rbase, __ffs(listed) - 1);
        const uint32_t r = rbase + __popc(below);
        const unsigned peers = __match_any_sync(listed, bin);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(P.bin_count + bin, (unsigned)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        const uint32_t slot = base + __popc(peers & ((1u << lane) - 1u));
        P.bin_list[(size_t)bin * P.bin_stride + slot] = r;
        if (P.ray_index) P.ray_index[i] = r;
        const uint4 *src = reinterpret_cast<const uint4 *>(&rec);
        uint4 *dst = reinterpret_cast<uint4 *>(P.rays_a + r);
#pragma unroll
        for (int k = 0; k < 4; k++) st_stream(dst + k, src[k]);
        src = reinterpret_cast<const uint4 *>(&rb);
        dst = reinterpret_cast<uint4 *>(P.rays_b + r);
#pragma unroll
        for (int k = 0; k < 5; k++) st_stream(dst + k, src[k]);
    } else if (in_range) {
        TaskOut o;
        o.first_hit = 0xffffffffu;
        o.steps = 0;
        o.flags = octant;
        o.n_hits = 0;
        *reinterpret_cast<uint4 *>(P.task_out + i) = *reinterpret_cast<const uint4 *>(&o);
    }
}

// ======================================================================================================
// Kernel 2 — the marching kernel (replaces SpaceRaytracer::trace_ray's loop, sr.rs:180-238, and the Rayon
// dispatch, renderer.rs:516-556): persistent warps, lane refill from the ray list.
//
// One iteration of the hot loop is, for every marching lane (no divergent branch up to the surface case):
//   State::step (raycast.rs:577-626)           select the axis with the smallest t_max, add t_delta, move the index
//   bounds (raycast.rs:265-274)                per-axis counters of the steps left inside the level: one sign test
//   SurfaceIter / VoxelSurfaceIter lookup      one dependent 2-byte load (4 bytes in a wide brick pool); bit 15 = nothing to see
//   count_step_should_stop (sr.rs:625-656)     step counter, log-domain upper bound of the transmittance
//   DepthIter span end (surface.rs:460-490)    Volumetric: thickness of the pending surface's span -> its hit record
//   visible surface (surface.rs:322-331,399)   a 64-byte hit record into the lane's chunk of the hit stream
// A lane parks when it has to change level (EnterBlock: Raycaster::within on the brick, raycast.rs:458-476; leaving
// the brick) or when its ray is finished; parked lanes are served together once `event_threshold` lanes wait.
// WIDE: u32 cells; BRICK_WIDE: u32 brick words (a wide brick pool).
// ======================================================================================================
template <bool VOLUMETRIC, bool WIDE, bool AUX, bool BRICK_WIDE>
__global__ void __launch_bounds__(WARPS_PER_BLOCK * 32, AUX ? 1 : MIN_BLOCKS_PER_SM)
trace_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    grid_dependency_sync();
    const DeviceScene &S = P.scene;
    const int lane = threadIdx.x & 31;
    constexpr float F_NEG_INF = -__builtin_huge_valf();
    constexpr int COUNTER_STATIC = 0x3fffffff;   // steps left along an axis the ray does not move on

    unsigned long long n_outer = 0, n_inner = 0, n_blocks = 0;

    // Cold per-ray state lives in shared memory, one column per thread, so that the registers of the marching loop
    // hold only what a DDA step touches; the level switches read what they need into short-lived locals.
    __shared__ double sh_d[13][WARPS_PER_BLOCK * 32];
    __shared__ uint32_t sh_w[13][WARPS_PER_BLOCK * 32];
    // Volumetric: the first 48 bytes of the pending surface's hit record (HitRecord tmx..flags), written when its span
    // closes
    __shared__ uint4 sh_stash[VOLUMETRIC ? 3 : 1][WARPS_PER_BLOCK * 32];
    const int tid = threadIdx.x;
#define COLD_D(k) sh_d[k][tid]
#define COLD_W(k) sh_w[k][tid]
#define STASH(k) sh_stash[k][tid]
    // doubles: 0-2 origin, 3-5 direction, 6 half_over_len, 7 t_to_abs, 8-10 outer t_max while inside a block, 11 outer last_t
    // words:   0 outer index (= the Space cube of the entered block), 1-3 outer step counters, 4 outer face, 5 outer valid,
    //          6 record index (HitRecord::task), 7 first hit, 8 sky octant, 9 palette offset of the entered block,
    //          10 log2(resolution) of it, 11 pending surface's log2(1 - alpha) bound, 12 task;
    //          double 12: the pending surface's entry t
    // State that the marching loop only touches at a surface, a level switch or a refill lives in shared memory too:
    // with it in registers the Volumetric variants spill at 96 registers.
    __shared__ double sh_t_scale[WARPS_PER_BLOCK * 32];
    __shared__ uint32_t sh_hits[3][WARPS_PER_BLOCK * 32];
    __shared__ unsigned long long sh_dbg[3][WARPS_PER_BLOCK * 32];
    unsigned long long &dbg_t0 = sh_dbg[0][tid], &dbg_passes = sh_dbg[1][tid], &dbg_rays = sh_dbg[2][tid];
    dbg_t0 = dbg_passes = dbg_rays = 0;
    if (P.debug_warp_times) {
        unsigned long long t0;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        dbg_t0 = t0;
    }

    // the ray list: bins in order, longest chords first
    __shared__ uint32_t s_bin_start[N_BINS + 1];
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int b = 0; b < N_BINS; b++) { s_bin_start[b] = acc; acc += P.bin_count[b]; }
        s_bin_start[N_BINS] = acc;
    }
    __syncthreads();
    const uint32_t n_listed = s_bin_start[N_BINS];
    (void)n_chunk_tasks;

    // ---- per-ray state (registers) ---------------------------------------------------------------------
    int st = ST_IDLE;
    double tmx = 0.0, tmy = 0.0, tmz = 0.0, last_t = 0.0;   // State::t_max, last_t_distance of the active level
    double tdx = 0.0, tdy = 0.0, tdz = 0.0;                 // t_delta (raycast.rs:769)
    double &t_scale = sh_t_scale[tid];   // 1 on the outer level, 1/resolution inside a block (surface.rs:385-386)
    t_scale = 1.0;
    uint32_t idx = 0;                    // linear index of the current cube (cells) / voxel (brick pool)
    int stx = 0, sty = 0, stz = 0;       // signed index strides of the active level
    int cx = 0, cy = 0, cz = 0;          // steps left inside the level along each axis (< 0: outside)
    int fcx = 0, fcy = 0, fcz = 0;       // the face entered by a step along each axis (from the direction's signs)
    int face = 0;                        // Face7 through which the current cube was entered
    uint32_t sbits = 0;                  // (sx+1) | (sy+1)<<2 | (sz+1)<<4
    bool valid = false, inner = false, need_advance = false, have_pending = false;
    // Upper bound of log2 of the ColorBuf transmittance (never below the exact value the compositing computes).
    // Once it is under -8 the ray is certainly finished (sr.rs:648-652); in the rare case that only the exact value is
    // under 1/256 the marcher runs on and the compositing cuts the ray's hits and steps back (HitRecord::steps).
    // count_step_should_stop is then ONE compare per step: steps > step_limit, with step_limit = 1000 (sr.rs:639-643)
    // until the bound says "opaque", 0 from then on.
    float L = 0.0f;
    uint32_t steps = 0, step_limit = 1000u;
    uint32_t &n_hits = sh_hits[0][tid];  // hit records of the current ray (consecutive slots of this lane's chunks)
    uint32_t &chunk_base = sh_hits[1][tid], &chunk_used = sh_hits[2][tid];   // this lane's chunk of the hit stream
    n_hits = 0;
    chunk_base = HIT_NONE;
    chunk_used = HIT_CHUNK;
    uint32_t ev_word = 0;
    AuxState<AUX> aux{};
    bool list_exhausted = false;         // warp-uniform: the ray list has run out (tail of the frame)

    // log-domain bound of one transmittance factor.  Exact factor (shade_hit): 1 - clamp(1 - (f32)pow(u, th)) with
    // u = 1 - alpha, i.e. <= u^th (1 + 2^-23) + 2^-24; with u^th >= 2^-8.5 that is <= u^th * 2^(3.3e-5).  l2a >= log2(u)
    // (host, rounded up); the f32 product and sum add < 2e-6.  A factor under 2^-8.5 makes the ray opaque by itself.
    auto bound_factor = [&](float p) {
        L = (p < -8.5f) ? F_NEG_INF : L + (p + 1e-4f);
        step_limit = (L < -8.0f) ? 0u : 1000u;
    };

    // State::step (raycast.rs:577-626) on the active level, select-based so that lanes stepping along different axes
    // stay converged.  Axis choice as the reference: x if t_max.x is strictly the smallest, else y if
    // t_max.y < t_max.z, else z.  Returns true if the new cube is outside the level (raycast.rs:265-274).
    auto advance = [&]() -> bool {
        const bool xy = tmx < tmy, xz = tmx < tmz, yz = tmy < tmz;
        const bool ax = xy & xz;
        const bool ay = !xy & yz;
        const bool axy = ax | ay;
        const double tm = ax ? tmx : (ay ? tmy : tmz);
        const double td = ax ? tdx : (ay ? tdy : tdz);
        const double nt = tm + td;
        last_t = tm;
        tmx = ax ? nt : tmx;
        tmy = ay ? nt : tmy;
        tmz = axy ? tmz : nt;
        idx += (uint32_t)(ax ? stx : (ay ? sty : stz));
        face = ax ? fcx : (ay ? fcy : fcz);
        cx -= ax ? 1 : 0;
        cy -= ay ? 1 : 0;
        cz -= axy ? 0 : 1;
        return (cx | cy | cz) < 0;
    };

    // The same step with one branch per axis instead of selects: a third of the instructions on the path taken.  For
    // the tail of a frame, when a warp is down to a few long rays and the length of the dependent instruction chain
    // of one step — not the number of issue slots — is what the frame waits for.
    auto advance_branchy = [&]() -> bool {
        if ((tmx < tmy) & (tmx < tmz)) {
            last_t = tmx; tmx = tmx + tdx; idx += (uint32_t)stx; face = fcx; cx -= 1;
            return cx < 0;
        } else if (tmy < tmz) {
            last_t = tmy; tmy = tmy + tdy; idx += (uint32_t)sty; face = fcy; cy -= 1;
            return cy < 0;
        } else {
            last_t = tmz; tmz = tmz + tdz; idx += (uint32_t)stz; face = fcz; cz -= 1;
            return cz < 0;
        }
    };

    // A slot of the lane's chunk of the hit stream for the ray's next record, or HIT_NONE once the stream is full.
    auto take_slot = [&]() -> uint32_t {
        if (chunk_used == HIT_CHUNK) {   // one atomic per HIT_CHUNK hits of this lane
            const uint32_t nb = atomicAdd(P.hit_counter, HIT_CHUNK);
            if (nb + HIT_CHUNK > P.hit_capacity) {   // (the capacity is a multiple of HIT_CHUNK)
                *P.overflow_flag = 1u;               // the host re-runs the frame with a larger buffer
                chunk_base = HIT_NONE;
            } else {
                // a ray's records are consecutive slots; the last slot of a chunk says where they continue
                if (chunk_base != HIT_NONE && n_hits != 0) P.hits[chunk_base + HIT_CHUNK - 1].next = nb;
                chunk_base = nb;
            }
            chunk_used = 0;
        }
        uint32_t slot = HIT_NONE;
        if (chunk_base != HIT_NONE) {
            slot = chunk_base + chunk_used;
            chunk_used++;
            if (n_hits == 0) COLD_W(7) = slot;
            n_hits++;
        }
        return slot;
    };

    // The whole 64-byte record: the caster state at the surface (q0-q2), the thickness of its span, the step counter.
    auto store_record = [&](uint32_t slot, uint4 q0, uint4 q1, uint4 q2, float thickness) {
        uint4 *dst = reinterpret_cast<uint4 *>(P.hits + slot);
        st_stream(dst, q0);
        st_stream(dst + 1, q1);
        st_stream(dst + 2, q2);
        st_stream(dst + 3, make_uint4(__float_as_uint(thickness), steps, COLD_W(6), HIT_NONE));
    };

    // A visible surface (surface.rs:322-331, 399-409).  Surface / Threshold: its hit record goes to the lane's chunk of
    // the hit stream at once.  Volumetric: the record waits in the lane's stash until a later step closes the surface's
    // span (surface.rs:467-476), possibly on the outer level after the block is left, and is written whole then; a
    // surface whose ray stops before its span closes is never shaded, and takes no slot.
    auto emit_surface = [&](uint32_t word) {
        uint32_t entry;   // palette entry of the surface, and what the transmittance bound needs of it
        float2 te;
        if (inner) {
            entry = COLD_W(9) + word;
            te = __ldg(S.pal_tab + entry);
        } else {
            const float4 t4 = __ldg(S.blk_tab + word);
            te = make_float2(t4.x, t4.y);
            entry = __float_as_uint(t4.z);
        }
        const uint4 q0 = make_uint4((uint32_t)__double2loint(tmx), (uint32_t)__double2hiint(tmx),
                                    (uint32_t)__double2loint(tmy), (uint32_t)__double2hiint(tmy));
        const uint4 q1 = make_uint4((uint32_t)__double2loint(tmz), (uint32_t)__double2hiint(tmz),
                                    (uint32_t)__double2loint(last_t), (uint32_t)__double2hiint(last_t));
        const uint4 q2 = make_uint4(entry, inner ? COLD_W(0) : idx, idx,
                                    (uint32_t)face | (inner ? (8u | (COLD_W(10) << 4)) : 0u));
        if constexpr (VOLUMETRIC) {
            STASH(0) = q0;
            STASH(1) = q1;
            STASH(2) = q2;
            COLD_W(11) = __float_as_uint(te.y);
            COLD_D(12) = last_t * t_scale;
            have_pending = true;
        } else {
            const uint32_t slot = take_slot();
            if (slot != HIT_NONE) store_record(slot, q0, q1, q2, 0.0f);
            if (P.transparency == AICB_TRANSPARENCY_THRESHOLD) {   // limit_alpha (graphics_options.rs:496-507)
                if (te.x > P.threshold) L = F_NEG_INF;
            } else {
                bound_factor(te.y);
            }
        }
    };

    // One step of the ray: advance, look at the cube / voxel, count, close the open span, classify.
    auto step = [&](auto lean) {
        bool left = false;
        if (need_advance) {
            if (!valid) {   // the iterator ends without an exit step (raycast.rs:245-249)
                st = inner ? ST_POP : ST_DONE;
                return;
            }
            if constexpr (decltype(lean)::value) left = advance_branchy(); else left = advance();
        }
        need_advance = true;
        uint32_t w = 0;
        if (!left) {
            if constexpr (WIDE) {
                if (!inner) {
                    const uint32_t cell = __ldg((const uint32_t *)S.cells + idx);   // id | kind<<16
                    w = (cell & 0x3fffu) | ((cell >> 2) & 0xc000u);                  // only ids < 16384 keep their bits here
                    ev_word = cell & 0xffffu;
                } else {
                    if constexpr (BRICK_WIDE) w = __ldg((const uint32_t *)S.bricks + idx);
                    else w = __ldg(S.bricks + idx);
                }
            } else {
                if constexpr (BRICK_WIDE) w = inner ? __ldg((const uint32_t *)S.bricks + idx) : __ldg((const uint16_t *)S.cells + idx);
                else w = __ldg((inner ? S.bricks : (const uint16_t *)S.cells) + idx);
            }
            if constexpr (AUX) { if (inner) aux.n_inner++; else aux.n_outer++; }
        }
        // count_step_should_stop (sr.rs:625-656): every TraceStep / DepthStep is counted before it is looked at
        steps += 1;
        if (steps > step_limit) { st = ST_DONE; return; }
        if constexpr (VOLUMETRIC) {
            if (have_pending) {   // DepthIter: this step's t ends the pending surface's span (surface.rs:460-490)
                const float th = fmaxf((float)((last_t * t_scale - COLD_D(12)) * COLD_D(7)), 0.0f);   // sr.rs:720-731
                const float pend_l2a = __uint_as_float(COLD_W(11));
                const uint32_t slot = take_slot();
                if (slot != HIT_NONE) store_record(slot, STASH(0), STASH(1), STASH(2), th);
                bound_factor(pend_l2a == F_NEG_INF ? F_NEG_INF : th * pend_l2a);
                have_pending = false;
            }
        }
        if (left) {   // exit step: TraceStep::Invisible at this t (surface.rs:296-301, 388-393)
            st = inner ? ST_POP : ST_DONE;
            return;
        }
        if (w & 0x8000u) return;   // nothing to see here
        if (!inner && (w & 0x4000u)) {   // TraceStep::EnterBlock (surface.rs:334-352)
            if constexpr (VOLUMETRIC) {
                // the buffered DepthStep::EnterBlock is counted after the flushed span (surface.rs:478-488)
                steps += 1;
                if (steps > step_limit) { st = ST_DONE; return; }
            }
            if constexpr (!WIDE) ev_word = w & 0x3fffu;
            st = ST_ENTER;
            return;
        }
        const uint32_t voxel = BRICK_WIDE ? w >> 16 : w;   // a brick word's palette index
        if constexpr (WIDE) emit_surface(inner ? voxel : ev_word);
        else emit_surface(inner ? voxel : (w & 0x3fffu));
    };

    for (;;) {
        dbg_passes++;
        // =========================== FINALIZE: hand the ray's result to the compositing ==================
        if (st == ST_DONE) {
            dbg_rays++;
            TaskOut o;
            o.first_hit = COLD_W(7);
            o.steps = steps;
            o.flags = COLD_W(8);
            o.n_hits = n_hits;
            *reinterpret_cast<uint4 *>(P.task_out + COLD_W(12)) = *reinterpret_cast<const uint4 *>(&o);
            if constexpr (AUX) { n_outer += aux.n_outer; n_inner += aux.n_inner; n_blocks += aux.n_blocks; }
            st = ST_IDLE;
        }
        // =========================== REFILL: idle lanes take the next rays of the list ====================
        {
            const unsigned idle = __ballot_sync(0xffffffffu, st == ST_IDLE);
            if (idle && !list_exhausted) {
                const int n = __popc(idle);
                uint32_t base = 0;
                const int leader = __ffs(idle) - 1;
                if (lane == leader) base = atomicAdd(P.task_counter, (unsigned)n);
                base = __shfl_sync(0xffffffffu, base, leader);
                if (st == ST_IDLE) {
                    const uint32_t k = base + __popc(idle & ((1u << lane) - 1u));
                    if (k >= n_listed) {
                        st = ST_EXHAUSTED;
                    } else {
                        int b = 0;
                        while (k >= s_bin_start[b + 1]) b++;
                        const uint32_t ri = __ldg(P.bin_list + (size_t)b * P.bin_stride + (k - s_bin_start[b]));
                        RayRecordA rec;
                        RayRecordB rb;
                        {
                            // A stays in L2 for the shading of the ray's hits; B is not read again (evict-first)
                            const uint4 *src = reinterpret_cast<const uint4 *>(P.rays_a + ri);
                            uint4 *dst = reinterpret_cast<uint4 *>(&rec);
#pragma unroll
                            for (int q = 0; q < 4; q++) dst[q] = ld_stream(src + q);
                            src = reinterpret_cast<const uint4 *>(P.rays_b + ri);
                            dst = reinterpret_cast<uint4 *>(&rb);
#pragma unroll
                            for (int q = 0; q < 5; q++) dst[q] = __ldcs(src + q);
                        }
                        const uint32_t task = rb.task;
                        COLD_W(6) = ri;
                        COLD_W(12) = task;
                        COLD_D(0) = rec.ox; COLD_D(1) = rec.oy; COLD_D(2) = rec.oz;
                        COLD_D(3) = rec.dx; COLD_D(4) = rec.dy; COLD_D(5) = rec.dz;
                        COLD_D(6) = rb.half_over_len;
                        COLD_D(7) = rec.t_to_abs;
                        COLD_W(7) = HIT_NONE;
                        COLD_W(8) = (rec.flags >> 12) & 7u;
                        tdx = rb.tdx; tdy = rb.tdy; tdz = rb.tdz;
                        tmx = rb.tmx; tmy = rb.tmy; tmz = rb.tmz; last_t = rb.last_t;
                        sbits = (rec.flags >> 6) & 0x3fu;
                        const int sx = (int)(sbits & 3u) - 1, sy = (int)((sbits >> 2) & 3u) - 1, sz = (int)((sbits >> 4) & 3u) - 1;
                        fcx = sx > 0 ? AICB_FACE_NX : AICB_FACE_PX;
                        fcy = sy > 0 ? AICB_FACE_NY : AICB_FACE_PY;
                        fcz = sz > 0 ? AICB_FACE_NZ : AICB_FACE_PZ;
                        stx = sx * (S.size[1] * S.size[2]); sty = sy * S.size[2]; stz = sz;
                        cx = sx > 0 ? S.size[0] - 1 - rb.rx : (sx < 0 ? rb.rx : COUNTER_STATIC);
                        cy = sy > 0 ? S.size[1] - 1 - rb.ry : (sy < 0 ? rb.ry : COUNTER_STATIC);
                        cz = sz > 0 ? S.size[2] - 1 - rb.rz : (sz < 0 ? rb.rz : COUNTER_STATIC);
                        idx = (uint32_t)((rb.rx * S.size[1] + rb.ry) * S.size[2] + rb.rz);   // as caster_begin
                        face = (int)(rec.flags & 7u);
                        valid = (rec.flags & 16u) != 0;
                        L = 0.0f;
                        step_limit = 1000u;
                        if (P.target.in_accum) {   // the layers in front may have made the ray opaque already
                            const float t0 = __ldg(&P.target.in_accum[P.task_base + task].w);
                            L = (t0 > 0.0f) ? __log2f(t0) + 1e-3f : F_NEG_INF;
                            step_limit = (L < -8.0f) ? 0u : 1000u;
                        }
                        steps = 0;
                        n_hits = 0;
                        have_pending = false;
                        inner = false;
                        t_scale = 1.0;
                        need_advance = false;
                        if constexpr (AUX) aux.n_outer = aux.n_inner = aux.n_blocks = 0;
                        st = ST_MARCH;
                    }
                }
                if (__any_sync(0xffffffffu, st == ST_EXHAUSTED)) list_exhausted = true;
            }
            if (__all_sync(0xffffffffu, st == ST_EXHAUSTED || st == ST_IDLE)) break;
        }
        // =========================== recursive_raycast (raycast.rs:458-476) + TraceStep::EnterBlock ======
        if (st == ST_ENTER) {
            if constexpr (AUX) aux.n_blocks++;
            const uint4 *bp = reinterpret_cast<const uint4 *>(S.blocks + ev_word);
            const uint4 b0 = __ldg(bp);
            const uint4 b1 = __ldg(bp + 1);
            const int bres = (int)(b0.x >> 8);
            Level in;
            in.lox = (int16_t)(b0.y & 0xffff); in.loy = (int16_t)(b0.y >> 16); in.loz = (int16_t)(b0.z & 0xffff);
            in.nx = (int)(b0.z >> 16); in.ny = (int)(b0.w & 0xffff); in.nz = (int)(b0.w >> 16);
            in.base = b1.x;
            const double fres = (double)bres;
            // the Space cube of this block, from its linear index
            const uint32_t nyz = (uint32_t)S.size[1] * (uint32_t)S.size[2];
            const uint32_t qx = idx / nyz, rem = idx - qx * nyz;
            const uint32_t qy = rem / (uint32_t)S.size[2], qz = rem - qy * (uint32_t)S.size[2];
            const int ccx = (int)qx + S.lo[0], ccy = (int)qy + S.lo[1], ccz = (int)qz + S.lo[2];
            Ray rr;
            rr.ox = COLD_D(0); rr.oy = COLD_D(1); rr.oz = COLD_D(2);
            rr.dx = COLD_D(3); rr.dy = COLD_D(4); rr.dz = COLD_D(5);
            rr.tdx = tdx; rr.tdy = tdy; rr.tdz = tdz;
            rr.half_over_len = COLD_D(6);
            rr.sx = (int)(sbits & 3u) - 1; rr.sy = (int)((sbits >> 2) & 3u) - 1; rr.sz = (int)((sbits >> 4) & 3u) - 1;
            Caster ic;
            bool ivalid;
            if (caster_begin(ic, rr, (rr.ox - (double)ccx) * fres, (rr.oy - (double)ccy) * fres, (rr.oz - (double)ccz) * fres, in,
                             &ivalid)) {
                COLD_D(8) = tmx; COLD_D(9) = tmy; COLD_D(10) = tmz; COLD_D(11) = last_t;
                COLD_W(0) = idx; COLD_W(1) = (uint32_t)cx; COLD_W(2) = (uint32_t)cy; COLD_W(3) = (uint32_t)cz;
                COLD_W(4) = (uint32_t)face; COLD_W(5) = valid ? 1u : 0u;
                COLD_W(9) = b1.y;
                COLD_W(10) = (uint32_t)(31 - __clz(bres));
                tmx = ic.tmx; tmy = ic.tmy; tmz = ic.tmz; last_t = ic.last_t;
                idx = ic.idx;
                face = ic.face;
                valid = ivalid;
                cx = rr.sx > 0 ? in.nx - 1 - ic.rx : (rr.sx < 0 ? ic.rx : COUNTER_STATIC);
                cy = rr.sy > 0 ? in.ny - 1 - ic.ry : (rr.sy < 0 ? ic.ry : COUNTER_STATIC);
                cz = rr.sz > 0 ? in.nz - 1 - ic.rz : (rr.sz < 0 ? ic.rz : COUNTER_STATIC);
                stx = rr.sx * (in.ny * in.nz); sty = rr.sy * in.nz; stz = rr.sz;
                inner = true;
                t_scale = recip_pow2(bres);
                need_advance = false;
            }
            st = ST_MARCH;
        }
        // =========================== back to the Space level ==============================================
        if (st == ST_POP) {
            tmx = COLD_D(8); tmy = COLD_D(9); tmz = COLD_D(10); last_t = COLD_D(11);
            idx = COLD_W(0); cx = (int)COLD_W(1); cy = (int)COLD_W(2); cz = (int)COLD_W(3);
            face = (int)COLD_W(4);
            valid = COLD_W(5) != 0;
            const int sx = (int)(sbits & 3u) - 1, sy = (int)((sbits >> 2) & 3u) - 1, sz = (int)((sbits >> 4) & 3u) - 1;
            stx = sx * (S.size[1] * S.size[2]); sty = sy * S.size[2]; stz = sz;
            inner = false;
            t_scale = 1.0;
            need_advance = true;
            st = ST_MARCH;
        }
        // =========================== MARCH ================================================================
        {
            const int n_off = __popc(__ballot_sync(0xffffffffu, st == ST_EXHAUSTED || (list_exhausted && st == ST_IDLE)));
            // How many waiting lanes end the marching loop.  While the list still has rays: `event_threshold`.  Once it is
            // exhausted the warp only drains: waiting for as many parked lanes as before would stall the rays the frame
            // is waiting for, serving every single park (a threshold of 1) makes a warp that still has all its rays —
            // every warp of a small shard, whose rays are all handed out in the first refill — run a full pass of the
            // level-switch code per step.  Half of the lanes that still have a ray is the compromise.
            int thr = (int)P.event_threshold;
            if (list_exhausted) {
                const int tail_div = (int)P.tail_divisor;
                thr = (32 - n_off) / (tail_div > 0 ? tail_div : 2);
                thr = thr < 1 ? 1 : (thr > (int)P.event_threshold ? (int)P.event_threshold : thr);
            }
            const unsigned live = __ballot_sync(0xffffffffu, st == ST_MARCH);
            if (list_exhausted && __popc(live) <= (int)P.refill_threshold) {
                // the tail: each of the few remaining rays runs to its next level switch on its own
                if (st == ST_MARCH) {
                    do { step(std::true_type{}); } while (st == ST_MARCH);
                }
            } else {
                for (;;) {
                    const unsigned marching = __ballot_sync(0xffffffffu, st == ST_MARCH);
                    if (!marching) break;
                    if (32 - __popc(marching) - n_off >= thr) break;   // enough lanes wait for the warp
                    if (st == ST_MARCH) step(std::false_type{});
                }
            }
        }
        __syncwarp();
    }

    if (P.debug_warp_times) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        unsigned long long rays = dbg_rays;
        for (int off = 16; off > 0; off >>= 1) rays += __shfl_down_sync(0xffffffffu, rays, off);
        if (lane == 0) {
            unsigned long long *d = P.debug_warp_times + 4 * (size_t)(blockIdx.x * WARPS_PER_BLOCK + (threadIdx.x >> 5));
            d[0] = dbg_t0; d[1] = t1; d[2] = dbg_passes; d[3] = rays;
        }
    }
    // the unused rest of this lane's chunk of the hit stream: never shaded
    if (chunk_base != HIT_NONE)
        for (uint32_t j = chunk_used; j < HIT_CHUNK; j++) P.hits[chunk_base + j].thickness = -2.0f;

    if constexpr (AUX) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            n_outer += __shfl_down_sync(0xffffffffu, n_outer, off);
            n_inner += __shfl_down_sync(0xffffffffu, n_inner, off);
            n_blocks += __shfl_down_sync(0xffffffffu, n_blocks, off);
        }
        if (lane == 0) {
            atomicAdd(P.counters + 1, n_outer);
            atomicAdd(P.counters + 2, n_inner);
            atomicAdd(P.counters + 5, n_blocks);
        }
    }
#undef COLD_D
#undef COLD_W
#undef STASH
}

// Position of a hit (hit.rs:92-101) from its record: Space cube, voxel, resolution, face, and the palette entry.
struct HitGeom {
    int cube[3];
    int voxel[3];
    int res;
    int face;
    uint32_t pal;
};
AICB_DEV void decode_hit(const DeviceScene &S, const HitRecord &h, HitGeom &g) {
    const uint32_t nz = (uint32_t)S.size[2], nyz = (uint32_t)S.size[1] * nz;
    const uint32_t qx = h.cell / nyz, rem = h.cell - qx * nyz;
    const uint32_t qy = rem / nz, qz = rem - qy * nz;
    g.cube[0] = (int)qx + S.lo[0]; g.cube[1] = (int)qy + S.lo[1]; g.cube[2] = (int)qz + S.lo[2];
    g.face = (int)(h.flags & 7u);
    if (h.flags & 8u) {
        const uint32_t id = S.wide_cells ? (__ldg((const uint32_t *)S.cells + h.cell) & 0xffffu)
                                         : ((uint32_t)__ldg((const uint16_t *)S.cells + h.cell) & 0x3fffu);
        const uint4 *bp = reinterpret_cast<const uint4 *>(S.blocks + id);
        const uint4 b0 = __ldg(bp);
        const uint32_t brick_off = __ldg(bp + 1).x;
        const uint32_t vny = b0.w & 0xffffu, vnz = b0.w >> 16;
        const uint32_t local = h.vidx - brick_off;
        const uint32_t vx = local / (vny * vnz), vrem = local - vx * (vny * vnz);
        const uint32_t vy = vrem / vnz, vz = vrem - vy * vnz;
        g.voxel[0] = (int)vx + (int)(int16_t)(b0.y & 0xffff);
        g.voxel[1] = (int)vy + (int)(int16_t)(b0.y >> 16);
        g.voxel[2] = (int)vz + (int)(int16_t)(b0.z & 0xffff);
        g.res = 1 << ((h.flags >> 4) & 15u);
    } else {
        g.voxel[0] = g.voxel[1] = g.voxel[2] = 0;
        g.res = 1;
    }
    g.pal = h.pal;
}

// RaycastStep::intersection_point (raycast.rs:409-439) of a hit, brought to Space coordinates (surface.rs:406-407):
// axis `a`, from the caster state the record holds, against the ray of the level the surface is on (the ray scaled
// into the block's voxel grid for an inner hit).  `ray` is the ray's origin and direction (RayRecordA's first six
// doubles).  One axis at a time, so that one axis of the ray is live at a time; select-based, as the face axis differs
// between the lanes of the shading kernel.
AICB_DEV double hit_point_axis(const HitRecord &h, const HitGeom &g, const double *ray, uint32_t rflags, int a) {
    const bool inner = (h.flags & 8u) != 0;
    const double cube = (double)g.cube[a];
    const double o = inner ? (__ldg(ray + a) - cube) * (double)g.res : __ldg(ray + a);
    const double base = (double)(inner ? g.voxel[a] : g.cube[a]);
    const double tm = a == 0 ? h.tmx : (a == 1 ? h.tmy : h.tmz);
    const double off = (tm - h.last_t) * __ldg(ray + 3 + a);
    const int s = (int)((rflags >> (6 + 2 * a)) & 3u) - 1;
    const double p_face = s < 0 ? base + 1.0 : base;
    const double p_other = base + ((s > 0) ? (1.0 - rclamp01(off)) : rclamp01(-off));
    const bool within = g.face == AICB_FACE_WITHIN;
    const double p = within ? o : (((g.face - 1) % 3 == a) ? p_face : (s == 0 ? o : p_other));
    return inner ? p * recip_pow2(g.res) + cube : p;
}

#ifdef AICB_SHADE_PHASES
// tools/shade_phases.py builds the library with this defined: clock64 cycles of the phases of shade_hit<LC_INTERP>,
// summed over a frame's hits (SHADE_PHASE_NAMES there).  The build the library ships has no trace of it.
__device__ unsigned long long g_shade_phase[10];
#define SHADE_PHASE(k)                                                                                                 \
    do {                                                                                                               \
        if constexpr (LC == LC_INTERP) {                                                                               \
            const long long t_ = clock64();                                                                            \
            ph_[k] = t_ - t0_;                                                                                         \
            t0_ = t_;                                                                                                  \
        }                                                                                                              \
    } while (0)
#else
#define SHADE_PHASE(k) do {} while (0)
#endif

// One hit record -> its ShadedHit (returned, not stored: resolve_kernel keeps it in shared memory, shade_kernel and
// bounce_resolve_kernel store it).  `illum_override` (LC_BOUNCE only): the illumination gathered by the hit's
// secondary rays; without it a Bounce frame lights the surface like Flat (surface.rs:171-176) and marks fully opaque
// surfaces (the only ones the bounce RNG is handed to, surface.rs:85-88) for bounce_select_kernel.
template <int LC>
AICB_DEV ShadedHit shade_hit(const TraceParams &P, const float *s_lut, const uint32_t i, const float *illum_override,
                             unsigned long long &texels) {
    const DeviceScene &S = P.scene;
    const bool volumetric = P.transparency == AICB_TRANSPARENCY_VOLUMETRIC;
    const bool have_fog = (P.fog != AICB_FOG_NONE) && P.include_sky;
    const float fog_blend = (P.fog == AICB_FOG_ABRUPT) ? 1.0f : (P.fog == AICB_FOG_COMPROMISE ? 0.5f : 0.0f);
#ifdef AICB_SHADE_PHASES
    long long ph_[7] = {0, 0, 0, 0, 0, 0, 0}, t0_ = clock64();
    struct Flush {
        long long *ph;
        __device__ ~Flush() {
            for (int k = 0; k < 7; k++) atomicAdd(&g_shade_phase[k], (unsigned long long)ph[k]);
        }
    } flush_{ph_};
#endif
    HitRecord h;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(P.hits + i);
        uint4 *dst = reinterpret_cast<uint4 *>(&h);
#pragma unroll
        for (int k = 0; k < 4; k++) dst[k] = ld_stream(src + k);
    }
    // everything the shading reads through the record is requested now, before any of it is needed
    const RayRecordA *rp = P.rays_a + h.task;
    const float4 col = __ldg(S.palette + 2 * (size_t)h.pal);
    const float4 emi = __ldg(S.palette + 2 * (size_t)h.pal + 1);
    const uint2 rmeta = __ldg(reinterpret_cast<const uint2 *>(&rp->t_to_view));   // t_to_view, flags
    const uint32_t rflags = rmeta.y;
    ShadedHit out;
    out.r = out.g = out.b = 0.0f;
    out.factor = -1.0f;
    out.next = h.next;
    out.steps = h.steps;
    out._pad[0] = out._pad[1] = 0;
    if (h.thickness < 0.0f) return out;   // an unused slot: skipped
    SHADE_PHASE(0);
    HitGeom g;
    decode_hit(S, h, g);
    SHADE_PHASE(1);
    float ca = col.w;
    float coeff = 1.0f;
    bool zeroed = false;
    if (volumetric) {
        const float thickness = h.thickness;
        if (thickness == 0.0f) {
            if (col.w == 1.0f) { coeff = 1.0f; }
            else { zeroed = true; ca = 0.0f; coeff = 0.0f; }
        } else if (col.w == 1.0f) {
            ca = 1.0f; coeff = 1.0f;        // 0^thickness == 0 exactly: alpha 1, (0-1)/(0-1) == 1
        } else if (col.w == 0.0f) {
            ca = 0.0f; coeff = thickness;   // 1^thickness == 1 exactly
        } else {
            const float unit_t = 1.0f - col.w;
            // the short path pays where the kernel's occupancy is its register count (LC_INTERP); resolve_kernel's
            // None / Flat frames measured 1.3 % slower with it inlined, so they keep the call
            const float depth_t = LC == LC_INTERP ? powf_exact(unit_t, thickness) : powf_libm(unit_t, thickness);
            ca = zo_clamped(1.0f - depth_t);
            const float k = (unit_t == 1.0f) ? thickness : (depth_t - 1.0f) / (unit_t - 1.0f);
            coeff = fmaxf(k, 0.0f);
        }
    }
    SHADE_PHASE(2);
    const float kc = ps_clamped(coeff);
    const float er = volumetric ? ps_mul(emi.x, kc) : emi.x, eg = volumetric ? ps_mul(emi.y, kc) : emi.y,
                eb = volumetric ? ps_mul(emi.z, kc) : emi.z;
    if (P.transparency == AICB_TRANSPARENCY_THRESHOLD) {  // limit_alpha (graphics_options.rs:496-507)
        if (ca > P.threshold) { ca = 1.0f; } else { zeroed = true; ca = 0.0f; }
    }
    if (ca == 0.0f && er == 0.0f && eg == 0.0f && eb == 0.0f) return out;   // nothing to see: the ray is not touched
    const double t_scale = recip_pow2(g.res);
    float tr = 1.0f - ca;
    float fa = -1.0f;
    if (have_fog) {  // distance_fog (sr.rs:745-768)
        float rel = (float)(h.last_t * t_scale) * __uint_as_float(rmeta.x);
        rel = rel < 0.0f ? 0.0f : (rel > 1.0f ? 1.0f : rel);
        const float fog_exponential = 1.0f - (LC == LC_INTERP ? expf_exact(-1.6f * rel) : expf_libm(-1.6f * rel));
        const float fudged = fog_exponential / 0.79810348f;
        const float p4 = (rel * rel) * (rel * rel);
        fa = zo_clamped(fudged * (1.0f - fog_blend) + p4 * fog_blend);
        tr = tr * (1.0f - fa);
    }
    SHADE_PHASE(3);
    const float cr = zeroed ? 0.0f : col.x, cg = zeroed ? 0.0f : col.y, cb = zeroed ? 0.0f : col.z;
    float i0 = 1.0f, i1 = 1.0f, i2 = 1.0f;
    const int face = g.face;
    if constexpr (LC == LC_BOUNCE) {
        // marked for bounce_select_kernel: the ray's RNG is only handed to fully opaque surfaces (surface.rs:85-88)
        if (ca == 1.0f) out._pad[0] = 1u;
    }
    if (LC == LC_BOUNCE && illum_override) {
        i0 = illum_override[0]; i1 = illum_override[1]; i2 = illum_override[2];
    } else if constexpr (LC == LC_FLAT || LC == LC_BOUNCE) {
        int x = g.cube[0], y = g.cube[1], z = g.cube[2];
        if (face != AICB_FACE_WITHIN) {
            const int dd = face >= AICB_FACE_PX ? 1 : -1;
            const int ax = (face - 1) % 3;
            if (ax == 0) x += dd; else if (ax == 1) y += dd; else z += dd;
        }
        uint32_t tx = 0;
        const uint32_t t = get_packed_light(S, x, y, z, tx);
        texels += tx;
        i0 = s_lut[t & 255]; i1 = s_lut[(t >> 8) & 255]; i2 = s_lut[(t >> 16) & 255];
    } else if constexpr (LC == LC_INTERP) {
        // the ray's origin and direction are read here, not with the record: loaded up front they stayed live
        // through the transmittance and fog and cost the kernel its occupancy
        const double *ray = reinterpret_cast<const double *>(rp);
        double ip[3];
#pragma unroll
        for (int a = 0; a < 3; a++) ip[a] = hit_point_axis(h, g, ray, rflags, a);
        SHADE_PHASE(4);
        uint32_t tx = 0;
        float il[3];
        interpolated_light(S, s_lut, P.lighting, g.cube[0], g.cube[1], g.cube[2], face, ip[0], ip[1], ip[2], il, &tx);
        SHADE_PHASE(5);
        i0 = il[0]; i1 = il[1]; i2 = il[2];
        texels += tx;
    }
    float orr = ps_mul(ps_mul(cr, i0), ca) + er;   // reflect + emission (color.rs:708-710)
    float og = ps_mul(ps_mul(cg, i1), ca) + eg;
    float ob = ps_mul(ps_mul(cb, i2), ca) + eb;
    if (fa >= 0.0f) {  // blend towards the sky sample of this ray (surface.rs:97-100)
        const int k = S.sky_kind ? (int)((rflags >> 12) & 7u) : 0;
        const float comp = 1.0f - fa;
        orr = ps_mul(orr, comp) + ps_mul(S.sky_colors[k][0], fa);
        og = ps_mul(og, comp) + ps_mul(S.sky_colors[k][1], fa);
        ob = ps_mul(ob, comp) + ps_mul(S.sky_colors[k][2], fa);
    }
    out.r = orr; out.g = og; out.b = ob; out.factor = tr;
    SHADE_PHASE(6);
    return out;
}

AICB_DEV void store_shaded(const TraceParams &P, const uint32_t i, const ShadedHit &s) {
    uint4 *outp = reinterpret_cast<uint4 *>(P.shaded + i);
    outp[0] = reinterpret_cast<const uint4 *>(&s)[0];
    outp[1] = reinterpret_cast<const uint4 *>(&s)[1];
}

// ======================================================================================================
// Kernel 3 of a frame that does not run resolve_kernel — shading: one thread per HitRecord, fully convergent, into
// the ShadedHit stream.  Everything about a surface that does not depend
// on the surfaces in front of it: its position (cube, voxel, face) and intersection point (raycast.rs:409-439,
// surface.rs:406-407) from the recorded caster state, apply_transmittance (sr.rs:720-740,
// raytracer_components.rs:215-258; Volumetric only), limit_alpha (graphics_options.rs:496-507), the invisibility
// test of Surface::to_light (surface.rs:78-82), compute_illumination (surface.rs:113-206), reflect + emission
// (color.rs:708-710), distance fog (sr.rs:745-768, surface.rs:97-100).  Output per hit: the outgoing light and the
// factor by which the surface multiplies the ray's transmittance (add_color_internal,
// raytracer_components.rs:87-92), or "skip".
// ======================================================================================================
// One wave of persistent blocks: 6 per SM (80 registers, no spills).  Measured on the C2 bench frame (H100 SXM, 400 W
// power limit): 0.236 ms against 0.27 ms for 8 blocks per SM at 90 registers, of which 5 were resident and 3 ran as a
// second wave.
constexpr int SHADE_BLOCKS_PER_SM = 6;
constexpr int SHADE_BLOCKS_PER_SM_INTERP = 8;
template <int LC> constexpr int shade_blocks_per_sm() { return LC == LC_INTERP ? SHADE_BLOCKS_PER_SM_INTERP : SHADE_BLOCKS_PER_SM; }
template <int LC>
__global__ void __launch_bounds__(128, shade_blocks_per_sm<LC>()) shade_kernel(const __grid_constant__ TraceParams P) {
    __shared__ float s_lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    grid_dependency_sync();
    __syncthreads();
    const DeviceScene &S = P.scene;
    uint32_t n = *P.hit_counter;
    if (n > P.hit_capacity) n = P.hit_capacity;
    unsigned long long texels = 0;
#ifdef AICB_SHADE_PHASES
    auto shade_one = [&](const uint32_t i) {
        const long long t0 = clock64();
        const ShadedHit sh = shade_hit<LC>(P, s_lut, i, nullptr, texels);
        const long long t1 = clock64();
        store_shaded(P, i, sh);
        const long long t2 = clock64();
        if (LC == LC_INTERP) {
            atomicAdd(&g_shade_phase[7], (unsigned long long)(t2 - t1));
            atomicAdd(&g_shade_phase[8], (unsigned long long)(t2 - t0));
            atomicAdd(&g_shade_phase[9], 1ull);
        }
    };
#else
    auto shade_one = [&](const uint32_t i) { store_shaded(P, i, shade_hit<LC>(P, s_lut, i, nullptr, texels)); };
#endif

    // The hit stream holds slots that are never shaded: the unused tail of each lane's last chunk.  Each warp scans its
    // slots 32 at a time, passes over the dead ones, and queues the live ones until it has 32 of them to shade
    // together.
    __shared__ uint32_t s_queue[4][64];
    uint32_t *queue = s_queue[threadIdx.x >> 5];
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    uint32_t queued = 0, base = warp * 32u;
    for (;;) {
        while (queued < 32u && base < n) {
            const uint32_t slot = base + lane;
            base += n_warps * 32u;
            bool live = false;
            // (no ray lists a dead slot, so none is read back: a chunk is full before its link is followed)
            if (slot < n) live = __ldg(&P.hits[slot].thickness) >= 0.0f;
            const unsigned m = __ballot_sync(0xffffffffu, live);
            if (live) queue[queued + __popc(m & ((1u << lane) - 1u))] = slot;
            queued += __popc(m);
            __syncwarp();
        }
        if (queued == 0u) break;
        const uint32_t take_n = queued < 32u ? queued : 32u;
        queued -= take_n;
        const uint32_t take = lane < take_n ? queue[queued + lane] : HIT_NONE;
        __syncwarp();
        if (take != HIT_NONE) shade_one(take);
    }
    // one atomic per warp: 150 K single-address atomics would cost more than the shading itself
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) texels += __shfl_down_sync(0xffffffffu, texels, off);
    if ((threadIdx.x & 31) == 0 && texels) atomicAdd(P.counters + 4, texels);
}

// ======================================================================================================
// LightingOption::Bounce (surface.rs:113-166, sr.rs:165-178).  A ray's RNG is only consulted at a fully opaque
// surface, and such a surface ends the ray (transmittance 0), so every ray bounces at most once: at its last
// accumulated hit.  A Bounce frame is therefore
//     gen -> march -> shade<LC_BOUNCE> (Flat light, marks fully opaque hits) -> bounce_select
//     -> `samples` x { bounce_gen -> gen -> march -> shade<LC_FLAT> -> encode (secondary mode: sums Rgb) }
//     -> bounce_resolve (re-shades the selected hits with the gathered illumination) -> encode.
// The secondary rays are ordinary rays of the same pipeline (trace_ray_impl(ray, .., include_sky = true,
// allow_ray_bounce = false): Flat lighting at their own hits) on a second set of per-frame streams.
// rand 0.10 SmallRng (xoshiro256++, SplitMix64 seeding) and rand_distr 0.6 UnitSphere are restated from their
// published algorithms (not under /root/reference): parity with the reference is unpinned, with the oracle exact.
// ======================================================================================================
AICB_DEV unsigned long long rotl64(unsigned long long x, int k) { return (x << k) | (x >> (64 - k)); }
AICB_DEV unsigned long long xoshiro_next(unsigned long long s[4]) {
    const unsigned long long result = rotl64(s[0] + s[3], 23) + s[0];
    const unsigned long long t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
    s[2] ^= t;
    s[3] = rotl64(s[3], 45);
    return result;
}
AICB_DEV void xoshiro_seed(unsigned long long s[4], unsigned long long state) {
    for (int pass = 0; pass < 2; pass++) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            state += 0x9e3779b97f4a7c15ull;
            unsigned long long z = state;
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            s[i] = z ^ (z >> 31);
        }
        if ((s[0] | s[1] | s[2] | s[3]) != 0ull) break;
        state = 0ull;   // an all-zero state is replaced by seed_from_u64(0)
    }
}
// Uniform::<f64>::new(-1.0, 1.0).sample(): 52 random mantissa bits in [1, 2), minus 1, times the scale 2, plus -1
AICB_DEV double uniform_m1_1(unsigned long long s[4]) {
    const unsigned long long bits = (xoshiro_next(s) >> 12) | 0x3ff0000000000000ull;
    return (__longlong_as_double((long long)bits) - 1.0) * 2.0 + (-1.0);
}

// Which hit, if any, a ray bounces at: the chain walk of encode_kernel (same stop rule) — the hit that ends the ray,
// if shade<LC_BOUNCE> marked it fully opaque.  Seeds the ray's RNG from its direction (sr.rs:165-178).
static __global__ void __launch_bounds__(128) bounce_select_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    grid_dependency_sync();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chunk_tasks) return;
    TaskOut o;
    *reinterpret_cast<uint4 *>(&o) = *reinterpret_cast<const uint4 *>(P.task_out + i);
    float T = 1.0f;
    if (P.target.in_accum) T = P.target.in_accum[P.task_base + i].w;
    uint32_t hi = o.first_hit, req = HIT_NONE;
    for (uint32_t hk = 0; hk < o.n_hits; hk++) {
        ShadedHit c;
        {
            const uint4 *src = reinterpret_cast<const uint4 *>(P.shaded + hi);
            reinterpret_cast<uint4 *>(&c)[0] = src[0];
            reinterpret_cast<uint4 *>(&c)[1] = src[1];
        }
        if (c.factor >= 0.0f) {
            T = T * c.factor;
            if (c._pad[0]) req = hi;
            if (T < (1.0f / 256.0f)) break;
        }
        hi = ((hi + 1u) & (HIT_CHUNK - 1u)) ? hi + 1u : c.next;
    }
    P.bounce_req[i] = req;
    P.bounce_sum[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(0u));
    if (req != HIT_NONE) {
        const RayRecordA *rp = P.rays_a + P.ray_index[i];   // (a ray with a hit was listed)
        const unsigned long long seed = (unsigned long long)__double_as_longlong(rp->dx) +
                                        (unsigned long long)__double_as_longlong(rp->dy) +
                                        (unsigned long long)__double_as_longlong(rp->dz);
        unsigned long long st[4];
        xoshiro_seed(st, seed);
        ulonglong2 *dst = reinterpret_cast<ulonglong2 *>(P.bounce_rng + 4 * (size_t)i);
        dst[0] = make_ulonglong2(st[0], st[1]);
        dst[1] = make_ulonglong2(st[2], st[3]);
    }
}

// The secondary ray of pass `bounce_pass` for every ray that bounces (surface.rs:131-153): from the intersection
// point, 1e-4 off the surface, towards normal + UnitSphere sample.
static __global__ void __launch_bounds__(128) bounce_gen_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    grid_dependency_sync();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chunk_tasks) return;
    const uint32_t req = P.bounce_req[i];
    if (req == HIT_NONE) return;
    const DeviceScene &S = P.scene;
    HitRecord h;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(P.hits + req);
        uint4 *dst = reinterpret_cast<uint4 *>(&h);
#pragma unroll
        for (int k = 0; k < 4; k++) dst[k] = src[k];
    }
    const RayRecordA *rp = P.rays_a + P.ray_index[i];
    HitGeom g;
    decode_hit(S, h, g);
    double ip[3];
#pragma unroll
    for (int a = 0; a < 3; a++) ip[a] = hit_point_axis(h, g, reinterpret_cast<const double *>(rp), rp->flags, a);
    double nrm[3] = {0.0, 0.0, 0.0};
    if (g.face != AICB_FACE_WITHIN) nrm[(g.face - 1) % 3] = g.face >= AICB_FACE_PX ? 1.0 : -1.0;
    unsigned long long st[4];
    {
        const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(P.bounce_rng + 4 * (size_t)i);
        const ulonglong2 a = src[0], b = src[1];
        st[0] = a.x; st[1] = a.y; st[2] = b.x; st[3] = b.y;
    }
    // rand_distr::UnitSphere (Marsaglia): reject until x1^2 + x2^2 < 1
    double x1, x2, sum;
    do {
        x1 = uniform_m1_1(st);
        x2 = uniform_m1_1(st);
        sum = x1 * x1 + x2 * x2;
    } while (sum >= 1.0);
    const double factor = 2.0 * sqrt(1.0 - sum);
    const double sph[3] = {x1 * factor, x2 * factor, 1.0 - 2.0 * sum};
    {
        ulonglong2 *dst = reinterpret_cast<ulonglong2 *>(P.bounce_rng + 4 * (size_t)i);
        dst[0] = make_ulonglong2(st[0], st[1]);
        dst[1] = make_ulonglong2(st[2], st[3]);
    }
    double *out = P.bounce_rays + 6 * (size_t)i;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        out[a] = ip[a] + nrm[a] * 0.0001;
        out[3 + a] = nrm[a] + sph[a];
    }
}

// Re-shades the hit each bouncing ray ends on with the mean of its secondary rays' light (surface.rs:161-165).
static __global__ void __launch_bounds__(128) bounce_resolve_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    __shared__ float s_lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = P.scene.tables[i];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_chunk_tasks) return;
    const uint32_t req = P.bounce_req[i];
    if (req == HIT_NONE) return;
    const float4 sum = P.bounce_sum[i];
    const float recip = ps_clamped(1.0f / (float)P.bounce_samples);   // Rgb * f32 clamps the scalar (color.rs:912-927)
    const float illum[3] = {ps_mul(sum.x, recip), ps_mul(sum.y, recip), ps_mul(sum.z, recip)};
    unsigned long long texels = 0;
    store_shaded(P, req, shade_hit<LC_BOUNCE>(P, s_lut, req, illum, texels));
}

// ======================================================================================================
// Per pixel, once the transmittance chain of each of its samples is known: finish (sr.rs:658-693: the sky;
// debug_pixel_cost), ColorBuf::mean of the 4 sub-samples in sample order (raytracer_components.rs:97-102), the
// encoder of draw_rgba (renderer.rs:287-291) and the stores.  `chain(k, o, lr, lg, lb, T, steps, sample_first)`
// yields sample k's accumulator after its hits (add_color_internal, raytracer_components.rs:87-92, with
// count_step_should_stop's opacity cut, sr.rs:648-652), its step count and the slot of its first visible surface.
// Returns the pixel's cubes_traced.
//
// TEX: the accumulator is RaytraceToTexture's Split (raytrace_to_texture.rs:922-977): ColorBuf, DepthBuf and the
// layer the pixel belongs to, stored as the colour and depth texels of trace_one (:622-683).  Split::add sets the layer
// of the first hit after which the ColorBuf is not OpacityCategory::Invisible (transmittance != 1).  Every hit
// multiplies the transmittance by a factor in [0, 1] (or sets it to 0: DebugOverrideRg), so once it is not 1 it
// never is again, and the first such hit can be found from the transmittance at the layer boundaries: the layer is Ui
// if the accumulator the world pass starts from (UI hits + backdrop, whose block data is the UI layer's,
// renderer.rs:242-252) has T != 1; otherwise this pass's layer if T != 1 after its hits; otherwise none.  P::paint
// (accum.rs:135-151) starts a fresh Split: depth +inf, layer World if the paint colour has T != 1.  The oracle
// (oracle_texture/aic_texture.cpp) applies the rule after each add it makes itself and after each layer's trace, and
// counts every layer whose trace raised the transmittance, so a case that broke the argument would show in the tests.
//
// TERM: the accumulator is the terminal's ColorCharacterBuf (all-is-cubes-desktop/src/terminal.rs:341-394): the
// ColorBuf, which alone decides opacity, and a CharacterBuf (text.rs:52-123) that every hit the colour gets is also
// added to.  CharacterBuf::add keeps the first Hit it is given, so per layer only the first hit that is a Hit matters:
// the first visible surface (its block), else Exception::Incomplete ("X"), else debug_pixel_cost's DebugOverrideRg
// (" "); the sky is ignored.  Without any of them a ray that counted a step (EnterSpace, sr.rs:629-637) has entered the
// space.  The backdrop adds " " after the UI layer's hits, and P::paint replaces the whole accumulator: text " ".  The
// UI pass hands the CharacterBuf on next to the ColorBuf (out_task_text); CharacterBuf::mean reduces the samples.
// ======================================================================================================
constexpr uint32_t TEX_NONE = 0, TEX_WORLD = 1, TEX_UI = 2;
// the target of a pixel-writing kernel (template): frames, aicb_render_layers_texture's texels, the terminal's pixels
constexpr int TGT_FRAME = 0, TGT_TEX = 1, TGT_TERM = 2;

// the Space block index of the cube a hit is in (the cell word's block field)
AICB_DEV int32_t hit_block(const TraceParams &P, uint32_t slot) {
    const DeviceScene &S = P.scene;
    const uint32_t cell = P.hits[slot].cell;
    return S.wide_cells ? (int32_t)(__ldg((const uint32_t *)S.cells + cell) & 0xffffu)
                        : (int32_t)((uint32_t)__ldg((const uint16_t *)S.cells + cell) & 0x3fffu);
}

AICB_DEV bool text_is_hit(int32_t t) { return t >= 0 || t <= AICB_TEXT_INCOMPLETE; }   // CharacterBuf State::Hit

template <bool TEX, bool TERM, class Chain>
AICB_DEV uint32_t finish_pixel(const TraceParams &P, const float *s_thr, const uint32_t i, const size_t out_index,
                               Chain &&chain) {
    const DeviceScene &S = P.scene;
    const uint32_t t0 = i * P.n_samples;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, aT = 0.f;
    uint32_t steps_total = 0;
    // Split::mean: the sub-samples' DepthBuf reduced by f64::min (a NaN start is what reduce() without an initial value
    // gives), the layer of the first sub-sample that has one
    double tex_depth = __longlong_as_double(0x7ff8000000000000ll);
    uint32_t tex_layer = TEX_NONE;
    double depth = D_INF;          // DepthBuf::mean = min over the sub-samples (accum.rs:284-297)
    uint32_t first_valid = 0xffffffffu;   // Position of the first surface hit: first sub-sample that has one
    int32_t text = AICB_TEXT_EMPTY;       // CharacterBuf of the pixel (text.rs:100-113 reduces the sub-samples)
    int2 term;                            // TERM: the pixel's CharacterBuf (text, layer), set by sample 0
    for (uint32_t k = 0; k < P.n_samples; k++) {
        TaskOut o;
        *reinterpret_cast<uint4 *>(&o) = *reinterpret_cast<const uint4 *>(P.task_out + t0 + k);
        float lr, lg, lb, T;
        uint32_t steps, sample_first;
        chain(k, o, lr, lg, lb, T, steps, sample_first);
        if (sample_first != 0xffffffffu && (P.target.out_depth || P.target.out_hit)) {
            const HitRecord *hr = P.hits + sample_first;   // Hit::t_distance = last_t / resolution (surface.rs:385-386)
            depth = fmin(depth, hr->last_t * recip_pow2(1 << ((hr->flags >> 4) & 15u)));
            if (first_valid == 0xffffffffu) first_valid = sample_first;
        }
        if (P.target.out_text) {
            // CharacterBuf::add (text.rs:84-98): the first hit of a block names it; Exception::Incomplete without one
            // is "X"; a ray that counted a step entered the space (sr.rs:628-637)
            int32_t tk = o.steps > 0 ? AICB_TEXT_ENTERED_SPACE : AICB_TEXT_EMPTY;
            if (sample_first != 0xffffffffu) {
                tk = hit_block(P, sample_first);
            } else if (o.steps > 1000u) {
                tk = AICB_TEXT_INCOMPLETE;
            }
            // CharacterBuf::mean (text.rs:100-113): the first sample that hit wins; entered only if all entered
            const bool ah = text >= 0 || text <= AICB_TEXT_INCOMPLETE, bh = tk >= 0 || tk <= AICB_TEXT_INCOMPLETE;
            if (k == 0) text = tk;
            else if (ah) {}
            else if (bh) text = tk;
            else if (text == AICB_TEXT_ENTERED_SPACE && tk == AICB_TEXT_ENTERED_SPACE) text = AICB_TEXT_ENTERED_SPACE;
            else text = AICB_TEXT_EMPTY;
        }
        if (P.include_sky) {  // the sky is an opaque hit at t = inf
            const int so = S.sky_kind ? (int)(o.flags & 7u) : 0;
            lr = lr + (S.sky_colors[so][0] * 1.0f) * T;
            lg = lg + (S.sky_colors[so][1] * 1.0f) * T;
            lb = lb + (S.sky_colors[so][2] * 1.0f) * T;
            T = T * (1.0f - 1.0f);
        }
        if (P.debug_pixel_cost) {  // ColorBuf::add for Exception::DebugOverrideRg (accum.rs:228-234)
            float kk = ps_clamped((float)steps);
            float red = ps_clamped(ps_mul(0.02f, kk) * 1.0f);
            float green = ps_clamped(ps_mul(0.002f, kk) * 1.0f);
            float rgba[4];
            colorbuf_to_rgba(lr, lg, lb, T, rgba);
            float lum = rgba[1] * 0.7152f + (rgba[0] * 0.2126f + rgba[2] * 0.0722f);
            lr = red; lg = green; lb = ps_clamped(lum * 0.2f);
            T = 0.0f;
        }
        if (P.target.has_backdrop) {   // Exception::Backdrop between the UI and the world (renderer.rs:458-466)
            lr = lr + P.target.backdrop[0] * T; lg = lg + P.target.backdrop[1] * T; lb = lb + P.target.backdrop[2] * T;
            T = T * P.target.backdrop[3];
        }
        if constexpr (TEX) {
            // DepthBuf::add (accum.rs:275-282): f64::min of the layer in front's depth and this layer's first surface
            double d = P.target.in_depth ? P.target.in_depth[P.task_base + t0 + k] : D_INF;
            if (sample_first != 0xffffffffu) {
                const HitRecord *hr = P.hits + sample_first;
                d = fmin(d, hr->last_t * recip_pow2(1 << ((hr->flags >> 4) & 15u)));
            }
            const float t_in = P.target.in_accum ? P.target.in_accum[P.task_base + t0 + k].w : 1.0f;
            uint32_t layer = t_in != 1.0f ? TEX_UI : (T != 1.0f ? P.target.tex_layer : TEX_NONE);
            if (P.target.has_no_world && !(T < (1.0f / 256.0f))) {   // P::paint: a fresh Split with the paint hit alone
                d = D_INF;
                layer = P.target.no_world[3] != 1.0f ? TEX_WORLD : TEX_NONE;
            }
            if (P.target.out_task_depth) P.target.out_task_depth[P.task_base + t0 + k] = d;
            tex_depth = fmin(tex_depth, d);
            if (tex_layer == TEX_NONE) tex_layer = layer;
        }
        if constexpr (TERM) {
            int2 c = P.target.in_text ? P.target.in_text[P.task_base + t0 + k] : make_int2(P.target.text_start, (int)TEX_NONE);
            if (!text_is_hit(c.x)) {   // CharacterBuf::add of this layer's hits, then the backdrop's
                if (sample_first != 0xffffffffu) c = make_int2(hit_block(P, sample_first), (int)P.target.tex_layer);
                else if (o.steps > 1000u) c.x = AICB_TEXT_INCOMPLETE;
                else if (P.debug_pixel_cost || P.target.has_backdrop) c.x = AICB_TEXT_BLANK;
                else if (o.steps > 0) c.x = AICB_TEXT_ENTERED_SPACE;
            }
            if (P.target.has_no_world && !(T < (1.0f / 256.0f))) c = make_int2(AICB_TEXT_BLANK, (int)TEX_NONE);   // P::paint
            if (P.target.out_task_text) P.target.out_task_text[P.task_base + t0 + k] = c;
            // CharacterBuf::mean (text.rs:96-108): the first sample that holds a Hit; EnteredSpace only if all entered
            if (k == 0 || (!text_is_hit(term.x) && text_is_hit(c.x))) term = c;
            else if (!text_is_hit(term.x))
                term.x = (term.x == AICB_TEXT_ENTERED_SPACE && c.x == AICB_TEXT_ENTERED_SPACE) ? AICB_TEXT_ENTERED_SPACE
                                                                                             : AICB_TEXT_EMPTY;
        }
        if (P.target.has_no_world && !(T < (1.0f / 256.0f))) {   // P::paint(NO_WORLD_TO_SHOW) replaces it (renderer.rs:474-477)
            lr = P.target.no_world[0]; lg = P.target.no_world[1]; lb = P.target.no_world[2]; T = P.target.no_world[3];
        }
        if (P.target.out_accum) P.target.out_accum[P.task_base + t0 + k] = make_float4(lr, lg, lb, T);
        if (P.bounce_mode == BOUNCE_SECONDARY) {
            // Rgba::from(light_accum_buf.inner).to_rgb() added to the surface's multi_ray_accum (surface.rs:158-160)
            if (P.bounce_req[t0 + k] != HIT_NONE) {
                float rgba[4];
                colorbuf_to_rgba(lr, lg, lb, T, rgba);
                float4 acc = P.bounce_sum[t0 + k];
                acc.x = acc.x + rgba[0]; acc.y = acc.y + rgba[1]; acc.z = acc.z + rgba[2];
                acc.w = __uint_as_float(__float_as_uint(acc.w) + steps);
                P.bounce_sum[t0 + k] = acc;
            }
            steps = 0;   // counted by the primary ray (RaytraceInfo + secondary_info, sr.rs:689-692)
        } else if (P.bounce_mode == BOUNCE_PRIMARY) {
            if (P.bounce_req[t0 + k] != HIT_NONE) steps += __float_as_uint(P.bounce_sum[t0 + k].w);
        }
        steps_total += steps;
        a0 = a0 + lr; a1 = a1 + lg; a2 = a2 + lb; aT = aT + T;
    }
    if (P.target.out_text) P.target.out_text[out_index] = text;
    float l0 = a0, l1 = a1, l2 = a2, tT = aT;
    if (P.n_samples == 4) { l0 = a0 / 4.0f; l1 = a1 / 4.0f; l2 = a2 / 4.0f; tT = aT / 4.0f; }
    if (P.target.out_srgb8) P.target.out_srgb8[out_index] = encode_srgb8(P, s_thr, l0, l1, l2, tT);
    if (P.target.out_colorbuf) P.target.out_colorbuf[out_index] = make_float4(l0, l1, l2, tT);
    if constexpr (TERM) {
        if (P.target.out_term) {   // ColorCharacterBuf::output (terminal.rs:355-366): post_process_color(Rgba::from(ColorBuf))
            float rgba[4], c[3];
            colorbuf_to_rgba(l0, l1, l2, tT, rgba);
            post_process_color(P, rgba, c);
            float2 *dst = reinterpret_cast<float2 *>(P.target.out_term + out_index);   // 24-byte pixels: 8-byte stores
            dst[0] = make_float2(c[0], c[1]);
            dst[1] = make_float2(c[2], rgba[3]);
            reinterpret_cast<int2 *>(dst)[2] = term;
        }
    }
    if constexpr (TEX) {
        if (P.target.out_rgba16f) {   // trace_one's colour (raytrace_to_texture.rs:643-661): the exposure of the pixel's layer
            const float e = tex_layer == TEX_UI ? P.target.tex_exposure[1] : (tex_layer == TEX_WORLD ? P.target.tex_exposure[0] : 1.0f);
            float a = 1.0f - tT;
            a = a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a);
            uint2 packed;
            packed.x = f16x2_texel(l0 * e, l1 * e);
            packed.y = f16x2_texel(l2 * e, a);
            P.target.out_rgba16f[out_index] = packed;
        }
        if (P.target.out_tex_depth) {
            // trace_one's depth (:663-674): clamp(0, 1) (NaN passes), depth_transform.transform_point3d_homogeneous
            // (0, 0, d) in euclid's term order, z / w as f32, the layer's sign (World +1, Ui or none -1)
            double d = tex_depth;
            if (d < 0.0) d = 0.0;
            if (d > 1.0) d = 1.0;
            const double *m = P.target.depth_m;
            const double z = ((0.0 * m[0] + 0.0 * m[1]) + d * m[2]) + m[3];
            const double w = ((0.0 * m[4] + 0.0 * m[5]) + d * m[6]) + m[7];
            P.target.out_tex_depth[out_index] = (float)(z / w) * (tex_layer == TEX_WORLD ? 1.0f : -1.0f);
        }
    } else if (P.target.out_rgba16f) {
        // ColorBuf::into_premultiplied_rgba (raytracer_components.rs:70-77) scaled by the exposure and rounded to
        // f16 as half::f16::from_f32 does (round to nearest even, overflow to infinity)
        float a = 1.0f - tT;
        a = a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a);   // clamp(0, 1): NaN passes through
        uint2 packed;
        packed.x = f16x2_texel(l0 * P.exposure, l1 * P.exposure);
        packed.y = f16x2_texel(l2 * P.exposure, a);
        P.target.out_rgba16f[out_index] = packed;
    }
    if (P.target.out_depth) P.target.out_depth[out_index] = depth;
    if (P.target.out_steps) P.target.out_steps[out_index] = steps_total;
    if (P.target.out_hit) {
        aicb_hit hh;
        if (first_valid != 0xffffffffu) {
            HitRecord hr;
            {
                const uint4 *src = reinterpret_cast<const uint4 *>(P.hits + first_valid);
#pragma unroll
                for (int q = 0; q < 4; q++) reinterpret_cast<uint4 *>(&hr)[q] = src[q];
            }
            HitGeom g;
            decode_hit(S, hr, g);
            hh.cube[0] = g.cube[0]; hh.cube[1] = g.cube[1]; hh.cube[2] = g.cube[2];
            hh.voxel[0] = g.voxel[0]; hh.voxel[1] = g.voxel[1]; hh.voxel[2] = g.voxel[2];
            hh.resolution = g.res;
            hh.face = g.face;
        } else {
            hh.cube[0] = hh.cube[1] = hh.cube[2] = -1;
            hh.voxel[0] = hh.voxel[1] = hh.voxel[2] = -1;
            hh.resolution = -1;
            hh.face = -1;
        }
        P.target.out_hit[out_index] = hh;
    }
    return steps_total;
}

// RaytraceInfo sum (renderer.rs:555) and the surface-hit counter: warp-reduce, one atomic per warp
AICB_DEV void count_pixels(const TraceParams &P, unsigned long long cubes_traced, unsigned long long n_hits) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        cubes_traced += __shfl_down_sync(0xffffffffu, cubes_traced, off);
        n_hits += __shfl_down_sync(0xffffffffu, n_hits, off);
    }
    if ((threadIdx.x & 31) == 0) {
        if (cubes_traced) atomicAdd(P.counters + 0, cubes_traced);
        if (n_hits) atomicAdd(P.counters + 3, n_hits);
    }
}

// ======================================================================================================
// Kernel 4 of a frame that does not run resolve_kernel — per pixel: the ray's transmittance chain over the ShadedHits
// that shade_kernel left, then finish_pixel.
// ======================================================================================================
// TGT: the texture targets of aicb_render_layers_texture or the terminal pixels of aicb_render_layers_terminal
// (finish_pixel); the instantiation other frames use (TGT_FRAME) carries neither.
constexpr uint32_t ENCODE_RUN = 4;
template <int TGT>
__global__ void __launch_bounds__(128) encode_kernel(const __grid_constant__ TraceParams P, uint32_t n_chunk_tasks) {
    constexpr bool TEX = TGT == TGT_TEX, TERM = TGT == TGT_TERM;
    __shared__ float s_thr[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_thr[i] = P.scene.tables[256 + i];
    grid_dependency_sync();
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;   // pixel task within the chunk
    const uint32_t n_pixels = n_chunk_tasks / P.n_samples;
    uint32_t px = 0, py = 0;
    size_t out_index = 0;
    const bool active = i < n_pixels && task_pixel<TEX>(P, P.task_base / P.n_samples + i, &px, &py, &out_index);
    unsigned long long cubes_traced = 0, n_hits = 0;
    if (active) {
        const uint32_t t0 = i * P.n_samples;
        cubes_traced = finish_pixel<TEX, TERM>(P, s_thr, i, out_index, [&](uint32_t k, const TaskOut &o, float &lr, float &lg, float &lb,
                                                               float &T, uint32_t &steps, uint32_t &sample_first) {
            lr = 0.f; lg = 0.f; lb = 0.f; T = 1.0f;
            if (P.target.in_accum) {   // what the layer in front left in the accumulator (renderer.rs:454-471)
                const float4 a = P.target.in_accum[P.task_base + t0 + k];
                lr = a.x; lg = a.y; lb = a.z; T = a.w;
            }
            steps = o.steps;
            sample_first = 0xffffffffu;
            uint32_t hi = o.first_hit;
            // the ray's consecutive slots, up to ENCODE_RUN at a time within a chunk: their colour and factor are
            // requested together (and the chunk's link with them), so a deep ray waits once per run, not once per hit
            for (uint32_t left = o.n_hits; left > 0u;) {
                const uint32_t chunk_last = hi | (HIT_CHUNK - 1u);
                const uint32_t run = min(left, min(ENCODE_RUN, chunk_last - hi + 1u));
                float4 f[ENCODE_RUN];
#pragma unroll
                for (uint32_t j = 0; j < ENCODE_RUN; j++)
                    if (j < run) f[j] = *reinterpret_cast<const float4 *>(P.shaded + hi + j);
                const bool to_end = hi + run > chunk_last;
                const uint32_t link = to_end ? P.shaded[chunk_last].next : HIT_NONE;
                bool cut = false;
#pragma unroll
                for (uint32_t j = 0; j < ENCODE_RUN; j++) {
                    if (j < run && !cut) {
                        const float4 c = f[j];
                        if (c.w >= 0.0f) {   // (a skipped surface leaves the ray untouched)
                            lr = lr + c.x * T; lg = lg + c.y * T; lb = lb + c.z * T;
                            T = T * c.w;
                            n_hits++;
                            if (sample_first == 0xffffffffu) sample_first = hi + j;
                            if (T < (1.0f / 256.0f)) {
                                // the reference stops at the first step it counts after this hit; the marcher, which
                                // only had an upper bound of T, may have gone further
                                const uint32_t cs = P.shaded[hi + j].steps;
                                if (steps > cs) steps = cs + 1;
                                cut = true;
                            }
                        }
                    }
                }
                if (cut) break;
                left -= run;
                hi = to_end ? link : hi + run;
            }
        });
    }
    count_pixels(P, cubes_traced, n_hits);
}

// ======================================================================================================
// Kernels 3+4 with None / Flat lighting (when the previous frame was shallow, launch_trace) — shading and compositing
// in one pass, tile by tile.
// One warp owns 32 consecutive tasks: one 8x4 tile of pixels, or with AntialiasingOption::Always 8 pixels x 4
// samples.  Neighbouring rays mostly meet the same or adjacent cubes, so shading their hits together turns the ray,
// palette, cell and light-texel loads into L1 hits, and no ShadedHit goes through global memory.  The warp works
// through its rays' hit lists in windows of RESOLVE_WINDOW slots held in shared memory:
//   list       an exclusive warp scan of the hits each lane has left places every lane's next slots in the window, in
//              ray order (the chunk links followed as encode_kernel does);
//   shade      the window's slots, 32 at a time, convergently (shade_hit; dead slots are skipped);
//   composite  every lane runs its own slots in order: light += c T, T *= factor, the cut at T < 1/256 and the step
//              restore.  A cut ray lists no more slots (its later surfaces cannot change the pixel).
// Then finish_pixel, one lane per pixel (with 4 samples the pixel's first lane reads its samples' accumulators back
// from shared memory, so the mean adds them in sample order as encode_kernel does).
// ======================================================================================================
constexpr uint32_t RESOLVE_WINDOW = 128;
// 4 resident blocks of 128 threads per SM = 128 registers per thread at most (the kernel needs about 80)
constexpr int RESOLVE_MIN_BLOCKS = 4;

template <int LC, int TGT>
__global__ void __launch_bounds__(128, RESOLVE_MIN_BLOCKS) resolve_kernel(const __grid_constant__ TraceParams P,
                                                                          uint32_t n_chunk_tasks) {
    static_assert(LC == LC_NONE || LC == LC_FLAT, "interpolated and Bounce lighting shade in shade_kernel");
    __shared__ float s_lut[256], s_thr[256];
    __shared__ float4 s_shaded[WARPS_PER_BLOCK][RESOLVE_WINDOW];   // r, g, b, factor (< 0: skip) of each window slot
    __shared__ uint32_t s_slot[WARPS_PER_BLOCK][RESOLVE_WINDOW];   // hit slot, later the lanes' first surface
    __shared__ uint32_t s_steps[WARPS_PER_BLOCK][RESOLVE_WINDOW];  // HitRecord::steps, later the lanes' step counts
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        s_lut[i] = P.scene.tables[i];
        s_thr[i] = P.scene.tables[256 + i];
    }
    grid_dependency_sync();
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    float4 *shaded = s_shaded[warp];
    uint32_t *slots = s_slot[warp], *hsteps = s_steps[warp];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;   // task within the chunk
    const uint32_t i = t / P.n_samples;                          // its pixel task
    uint32_t px = 0, py = 0;
    size_t out_index = 0;
    const bool active = t < n_chunk_tasks &&
                        task_pixel<TGT == TGT_TEX>(P, P.task_base / P.n_samples + i, &px, &py, &out_index);
    float lr = 0.f, lg = 0.f, lb = 0.f, T = 1.0f;
    uint32_t steps = 0, sample_first = 0xffffffffu, hi = HIT_NONE, left = 0;
    if (active) {
        TaskOut o;
        *reinterpret_cast<uint4 *>(&o) = *reinterpret_cast<const uint4 *>(P.task_out + t);
        if (P.target.in_accum) {   // what the layer in front left in the accumulator (renderer.rs:454-471)
            const float4 a = P.target.in_accum[P.task_base + t];
            lr = a.x; lg = a.y; lb = a.z; T = a.w;
        }
        steps = o.steps;
        hi = o.first_hit;
        left = o.n_hits;
    }
    unsigned long long texels = 0, n_hits = 0;
    for (;;) {
        // list: this lane's slots go to [first, first + take) of the window
        uint32_t incl = left;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, off);
            if ((int)lane >= off) incl += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        if (total == 0u) break;
        const uint32_t first = incl - left;
        const uint32_t take = first >= RESOLVE_WINDOW ? 0u : min(left, RESOLVE_WINDOW - first);
        const uint32_t listed = min(total, RESOLVE_WINDOW);
        // consecutive slots up to the end of the chunk (chunks are HIT_CHUNK-aligned), then the chunk's link: one
        // dependent load per chunk, requested before the run's stores
        for (uint32_t j = 0; j < take;) {
            const uint32_t chunk_last = hi | (HIT_CHUNK - 1u);
            const uint32_t run = min(take - j, chunk_last - hi + 1u);
            const bool to_end = hi + run > chunk_last;
            const uint32_t link = to_end ? __ldg(&P.hits[chunk_last].next) : HIT_NONE;
            for (uint32_t q = 0; q < run; q++) slots[first + j + q] = hi + q;
            j += run;
            hi = to_end ? link : hi + run;
        }
        left -= take;
        __syncwarp();
        // shade
        for (uint32_t b = 0; b < listed; b += 32u) {
            const uint32_t j = b + lane;
            if (j < listed) {
                const ShadedHit c = shade_hit<LC>(P, s_lut, slots[j], nullptr, texels);
                shaded[j] = make_float4(c.r, c.g, c.b, c.factor);
                hsteps[j] = c.steps;
            }
        }
        __syncwarp();
        // composite
        for (uint32_t j = first; j < first + take; j++) {
            const float4 c = shaded[j];
            if (c.w >= 0.0f) {   // (a skipped surface leaves the ray untouched)
                lr = lr + c.x * T; lg = lg + c.y * T; lb = lb + c.z * T;
                T = T * c.w;
                n_hits++;
                if (sample_first == 0xffffffffu) sample_first = slots[j];
                if (T < (1.0f / 256.0f)) {
                    // the reference stops at the first step it counts after this hit; the marcher, which only had an
                    // upper bound of T, may have gone further
                    if (steps > hsteps[j]) steps = hsteps[j] + 1;
                    left = 0;
                    break;
                }
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) texels += __shfl_down_sync(0xffffffffu, texels, off);
    if (lane == 0 && texels) atomicAdd(P.counters + 4, texels);

    // finish: the accumulators of the warp's tasks through shared memory to their pixel's first lane
    shaded[lane] = make_float4(lr, lg, lb, T);
    hsteps[lane] = steps;
    slots[lane] = sample_first;
    __syncwarp();
    unsigned long long cubes_traced = 0;
    if (active && t % P.n_samples == 0u) {
        cubes_traced = finish_pixel<TGT == TGT_TEX, TGT == TGT_TERM>(
            P, s_thr, i, out_index, [&](uint32_t k, const TaskOut &, float &r, float &g, float &b, float &tr,
                                        uint32_t &st, uint32_t &sf) {
            const float4 a = shaded[lane + k];
            r = a.x; g = a.y; b = a.z; tr = a.w;
            st = hsteps[lane + k];
            sf = slots[lane + k];
        });
    }
    count_pixels(P, cubes_traced, n_hits);
}

#endif  // __CUDACC__

}  // namespace aicb
