/*
 * aicb200.h — C ABI of libaicb200.so: the H100-native (sm_90a) replacement for the
 * per-pixel voxel raytracer of kpreid/all-is-cubes, behind the reference's own
 * HeadlessRenderer / Camera / SpaceRaytracer surface.
 *
 * Every entry point cites the reference interface it replaces (paths relative to the
 * reference checkout, commit 7ab02ee1).  All structs are plain data; all pointers in are
 * borrowed for the duration of the call only; all pointers out are caller-allocated with
 * explicit lengths.  Nothing throws or aborts across this boundary: errors are status codes
 * plus aicb_last_error().
 *
 * There is NO CPU fallback.  Every compute entry point fails with AICB_ERR_CUDA when no
 * compute capability 9.0 device (H100) is available.
 */
#ifndef AICB200_H
#define AICB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AICB_ABI_VERSION 28

typedef enum aicb_status {
    AICB_OK = 0,
    AICB_ERR_INVALID = 1,     /* bad argument / length mismatch (the reference panics: renderer.rs:193-197) */
    AICB_ERR_OOM = 2,         /* cudaMalloc failed  -> Flaws::OUT_OF_MEMORY (flaws.rs) */
    AICB_ERR_CUDA = 3,        /* no device, launch failure, lost GPU (lib.rs:53 "TODO: lost GPU") */
    AICB_ERR_UNSUPPORTED = 4, /* an option value this build does not implement */
    AICB_ERR_BUSY = 5,        /* aicb_render_finish for a scene whose frame is not the context's last one */
    AICB_ERR_RETRY = 6        /* asynchronous render only: the frame's hit stream overflowed its device buffer; the
                                 buffer has been enlarged, issue the same render again (the synchronous entry points
                                 retry internally) */
} aicb_status;

/* ---------------------------------------------------------------------------------------------
 * Plain-data mirrors of reference types
 * ------------------------------------------------------------------------------------------- */

/* GridAab (all-is-cubes-base/src/math/grid_aab.rs): lower corner + size. */
typedef struct aicb_aab {
    int32_t lower[3];
    uint32_t size[3];
} aicb_aab;

/* Evoxel (all-is-cubes/src/block/eval/voxel_storage.rs:41-60): non-premultiplied linear RGBA reflectance + RGB
 * emission, and `flags` (selectable, collision). 32 bytes. */
typedef struct aicb_voxel {
    float rgba[4];
    float emission[3];
    uint32_t flags;                /* AICB_VOXEL_*; other bits are ignored */
} aicb_voxel;
/* Evoxel::selectable == false (voxel_storage.rs:57).  Zero, the default, is selectable.  Only the cursor reads it. */
#define AICB_VOXEL_NOT_SELECTABLE 1u
/* Evoxel::collision == BlockCollision::None (voxel_storage.rs:60).  Zero, the default, is BlockCollision::Hard
 * (DEFAULT_FOR_FROM_COLOR, attributes.rs:527).  Only aicb_step_bodies reads it. */
#define AICB_VOXEL_NO_COLLISION 2u

/* Face7 (all-is-cubes-base/src/math/face.rs:105). */
enum { AICB_FACE_WITHIN = 0, AICB_FACE_NX = 1, AICB_FACE_NY = 2, AICB_FACE_NZ = 3,
       AICB_FACE_PX = 4, AICB_FACE_PY = 5, AICB_FACE_PZ = 6 };

/* One entry of Space::block_data() as the raytracer sees it: TracingBlock (sr.rs:569-587)
 * = Evoxels (voxel_storage.rs:190-209).  `indices == NULL` means Evoxels::One(palette[0]).
 * Otherwise `indices` holds one u16 palette index per voxel of `voxel_bounds`, Z-major
 * (vol.rs:1013-1018: ((x-lx)*size_y + (y-ly))*size_z + (z-lz)); voxel_bounds may be smaller
 * than resolution^3 (voxel_storage.rs:176-178) but must lie inside [0,resolution)^3.
 * `is_air` is TracingCubeData::always_invisible (sr.rs:547).
 * A palette may have up to 65536 entries (VoxelIndex is u16, voxel_storage.rs:32), duplicates and
 * unused entries included; more is AICB_ERR_UNSUPPORTED.  A scene whose blocks all have at most
 * 32768 entries keeps 2 bytes per voxel on the device; the first block with more makes it keep 4
 * (aicb_scene_device_bytes), until aicb_scene_fill_uniform replaces its table.
 * The `light_*` members are EvaluatedBlock derived data (block/eval/derived.rs:33-80) read
 * only by the light-propagation path (space/light/updater.rs:760-884). */
typedef struct aicb_block_desc {
    uint8_t resolution;            /* 1,2,4,...,128 (resolution.rs:18-27) */
    uint8_t is_air;
    uint8_t light_opaque_faces;    /* bit (face-1) set if EvaluatedBlock::opaque()[face], NX..PZ */
    uint8_t light_visible;         /* EvaluatedBlock::visible_or_animated() */
    aicb_aab voxel_bounds;
    const uint16_t *indices;       /* NULL => single voxel */
    size_t n_indices;
    const aicb_voxel *palette;
    size_t n_palette;
    float light_face_colors[6][4]; /* EvaluatedBlock::face7_color(face), NX..PZ */
    float light_color[4];          /* EvaluatedBlock::color() */
    float light_emission[3];       /* EvaluatedBlock::light_emission() */
    uint32_t flags;                /* AICB_BLOCK_*; other bits are ignored */
} aicb_block_desc;
/* BlockAttributes::selectable == false (attributes.rs:389).  Zero, the default, is selectable; an is_air block is never
 * selectable, whatever its flags (AIR_ATTRIBUTES, block/eval/evaluated.rs:419-421).  Only the cursor reads it. */
#define AICB_BLOCK_NOT_SELECTABLE 1u

/* Sky (all-is-cubes/src/space/sky.rs:16-21). kind 0 = Uniform(colors[0]), 1 = Octants.
 * Octant index = (x>=0)<<2 | (y>=0)<<1 | (z>=0)  (sky.rs:36-39). */
typedef struct aicb_sky {
    uint32_t kind;
    float colors[8][3];
} aicb_sky;

/* What SpaceRaytracer::new (sr.rs:64-88) snapshots from space::Read:
 * bounds, per-cube block index (Space::contents, Z-major), per-cube PackedLight texels
 * (light/data.rs:162 as_texel: r,g,b,status; NULL => LightPhysics::None => PackedLight::ONE,
 * space.rs:1241-1246), the block table and the sky. */
typedef struct aicb_scene_desc {
    aicb_aab bounds;
    const uint16_t *block_ids;     /* volume entries */
    const uint8_t (*light)[4];     /* volume texels or NULL */
    const aicb_block_desc *blocks;
    size_t n_blocks;
    aicb_sky sky;
    uint8_t light_max_distance;    /* LightPhysics::Rays{maximum_distance} (space/physics.rs:94-104); 0 = None */
    uint8_t _pad[7];
} aicb_scene_desc;

/* Camera as the raytracer consumes it: Camera::project_ndc_into_world (camera_struct.rs:238-257)
 * needs only inverse_projection_view (euclid Transform3D, row-vector convention, m11..m44 in
 * row-major order), the framebuffer size (viewport.rs:104-113) and exposure
 * (camera_struct.rs:376-382).  aicb_camera_look_at()/aicb_camera_from_view() below build it
 * exactly as Camera::compute_matrices (camera_struct.rs:387-416) does. */
typedef struct aicb_camera {
    double inverse_projection_view[16];
    uint32_t fb_width, fb_height;
    float exposure;
    uint32_t _pad;
} aicb_camera;

enum { AICB_FOG_NONE = 0, AICB_FOG_ABRUPT = 1, AICB_FOG_COMPROMISE = 2, AICB_FOG_PHYSICAL = 3 };
enum { AICB_LIGHT_NONE = 0, AICB_LIGHT_FLAT = 1, AICB_LIGHT_COARSE = 2, AICB_LIGHT_LINEAR = 3,
       AICB_LIGHT_SMOOTHSTEP = 4, AICB_LIGHT_BOUNCE = 5 /* secondary Lambertian rays (surface.rs:113-166); needs aicb_options::bounce_samples */ };
enum { AICB_TRANSPARENCY_SURFACE = 0, AICB_TRANSPARENCY_VOLUMETRIC = 1, AICB_TRANSPARENCY_THRESHOLD = 2 };
enum { AICB_TONE_CLAMP = 0, AICB_TONE_REINHARD = 1 };

/* The GraphicsOptions fields that affect pixels (graphics_options.rs:28-150). */
typedef struct aicb_options {
    uint8_t fog;
    uint8_t lighting_display;
    uint8_t transparency;
    uint8_t antialiasing_always;   /* AntialiasingOption::Always => 4 fixed sub-samples (renderer.rs:426-444) */
    uint8_t tone_mapping;
    uint8_t debug_pixel_cost;
    uint8_t include_sky;           /* trace_ray's include_sky argument (sr.rs:113-120); renders use 1 */
    uint8_t bounce_samples;        /* LightingOption::Bounce { samples } (graphics_options.rs:464-467); >= 1 with Bounce */
    float transparency_threshold;  /* TransparencyOption::Threshold(t) */
    float maximum_intensity;       /* +inf disables tone mapping (graphics_options.rs:352-357) */
    double view_distance;          /* repaired to [1, 10000] by the caller (graphics_options.rs:194-198) */
} aicb_options;

/* Row-strip sharding of one frame across ranks (SURVEY §8(e)): rows are cut into strips of
 * `strip_rows`; strip s belongs to shard (s % count).  count = 1 renders everything. */
typedef struct aicb_shard {
    uint32_t strip_rows;
    uint32_t index;
    uint32_t count;
} aicb_shard;

/* ImageInfo / RaytraceInfo (renderer.rs:609-646, sr.rs:520-522) plus device timing. */
typedef struct aicb_render_info {
    uint64_t cubes_traced;         /* RaytraceInfo::cubes_traced, summed over all rays */
    uint64_t rays;                 /* primary rays traced (pixels * samples) */
    uint64_t algorithmic_bytes;    /* SURVEY §8(d) formula, from device counters */
    uint64_t counters[6];          /* outer steps, inner steps, surface hits, light texels, blocks entered, pixels */
    float kernel_ms;               /* CUDA-event duration of the whole frame (all kernels) on its stream */
    uint16_t flaws;                /* Flaws bits (flaws.rs:20-91) */
    uint16_t ray_order;            /* 1: the marching kernel took the frame's rays in order of the steps their tiles took
                                      in the context's previous frame, of the same scene, camera view, size, samples and
                                      shard (a scheduling choice only: the outputs are the same either way); 0: in order
                                      of their chords through the Space */
    float stage_ms[4];             /* the frame's kernels (first chunk): ray generation, marching, shading, encode;
                                      where shading and encode ran as one kernel (LightingOption::None / Flat, most
                                      frames) [2] is its time and [3] is 0 */
} aicb_render_info;

/* CharacterBuf states (raytracer/text.rs:52-123) of aicb_render_text and aicb_render_layers_terminal: a value >= 0 is
 * the block index (Space palette index) of the first block hit; the caller maps it to that block's string like
 * TracingBlock's D::from_block does.  AICB_TEXT_BLANK comes from aicb_render_layers_terminal only. */
#define AICB_TEXT_ENTERED_SPACE (-1) /* the ray entered the Space's bounds but hit nothing: " " */
#define AICB_TEXT_EMPTY (-2)         /* the ray never entered the Space: "." */
#define AICB_TEXT_INCOMPLETE (-3)    /* Exception::Incomplete (step cap) before any hit: "X" */
#define AICB_TEXT_BLANK (-4)         /* a hit that names no block (backdrop, NO_WORLD_TO_SHOW paint, debug_pixel_cost): " " */

/* Per-pixel hit record: Position of the first non-exception Hit (hit.rs:92-101):
 * cube xyz, voxel xyz, resolution, face; all -1 when the ray hit nothing. */
typedef struct aicb_hit {
    int32_t cube[3];
    int32_t voxel[3];
    int32_t resolution;
    int32_t face;
} aicb_hit;

typedef struct aicb_ctx aicb_ctx;     /* one CUDA device + stream */
typedef struct aicb_scene aicb_scene; /* device-resident flattened Space */

/* ---------------------------------------------------------------------------------------------
 * Context
 * ------------------------------------------------------------------------------------------- */
uint32_t aicb_abi_version(void);
/* device_id < 0 selects the current device. Fails with AICB_ERR_CUDA if there is no GPU. */
aicb_status aicb_ctx_create(int device_id, aicb_ctx **out);
void aicb_ctx_destroy(aicb_ctx *);
/* aicb_render_info::stage_ms needs up to five event records per frame; on by default, off for callers that only want frames. */
aicb_status aicb_ctx_stage_timing(aicb_ctx *, int enable);
/* The CUDA device the context was created on (a device_id of -1 resolved to the device current then); -1 for NULL. */
int aicb_ctx_device(const aicb_ctx *);
/* Thread-local message for the last failing call on this thread. Never NULL. */
const char *aicb_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * Block evaluation: the light fields of EvaluatedBlock's derived data
 * ------------------------------------------------------------------------------------------- */
/* compute_derived (block/eval/derived.rs:80-216) of one block's voxels, the fields aicb_block_desc::light_* take. */
typedef struct aicb_block_light {
    float face_colors[6][4];   /* NX..PZ, what aicb_block_desc::light_face_colors takes */
    float color[4];
    float emission[3];
    uint8_t opaque_faces;      /* bit (face-1), as light_opaque_faces */
    uint8_t visible;
    uint8_t _pad[2];
} aicb_block_light;
/* == compute_derived (block/eval/derived.rs:80-216) for the light fields; reads only the voxel fields of descs.
 * A single voxel (indices == NULL, or resolution 1) gives its own colour and emission.  Any other block is traced on the
 * context's device: trace_for_eval (raytracer_components.rs:174-200) from every voxel face of the data bounds' six
 * sides, summed per face in iproduct!'s order, with the reference's f32 arithmetic (no contraction, the correctly
 * rounded powf).  `visible` is Derived::visible; EvaluatedBlock::visible_or_animated, which light_visible is, also
 * holds for blocks with an animation hint, which the caller ORs in.  is_air plays no part.
 * Blocks, runs on the context's stream after its queued work, and writes `out` only if it succeeds.  n == 0 does
 * nothing.  AICB_ERR_INVALID: a NULL pointer with n > 0, a block scene creation rejects (its status, so also
 * AICB_ERR_UNSUPPORTED for a palette over 65536 entries), or a colour or emission sum that is NaN (or negative) where
 * the reference's Rgb::try_from(..).expect(..) panics, with the block's position in aicb_last_error. */
aicb_status aicb_derive_block_light(aicb_ctx *, const aicb_block_desc *descs, size_t n, aicb_block_light *out);

/* ---------------------------------------------------------------------------------------------
 * update(): replaces SpaceRaytracer::new / UpdatingSpaceRaytracer::update
 * (sr.rs:64-88, updating.rs:107-172). The library copies everything before returning.
 * ------------------------------------------------------------------------------------------- */
aicb_status aicb_scene_create(aicb_ctx *, const aicb_scene_desc *, aicb_scene **out);
/* SpaceChange::CubeBlock / CubeLight (space.rs:1062-1100): light may be NULL to leave light alone. */
aicb_status aicb_scene_update_cubes(aicb_scene *, const int32_t (*cubes)[3], const uint16_t *block_ids,
                                    const uint8_t (*light)[4], size_t n);
/* SpaceChange::CubeBlock (and CubeLight) for every cube of `region`: the box form of aicb_scene_update_cubes, for a host
 * that filled a box (Space::fill, fill_uniform over a region, SpaceTransaction::filling).  block_ids: Z-major within
 * `region` (as Vol and interior_iter order them: z fastest), one entry per cube; NULL: every cube takes `uniform_id`.
 * light: Z-major within `region`, or NULL to leave the texels alone (ignored on a scene without a light volume, as
 * aicb_scene_update_cubes ignores it).  Nothing is built per cube on the host: the arrays go to the device as they are
 * (2 + 4 bytes per cube; a uniform fill uploads no ids) and the cells are encoded there, 16 bytes per store.  The light
 * update queue and the set of changed cubes are not touched.  Queued on the context's stream and ordered like
 * aicb_scene_update_cubes.  AICB_ERR_INVALID, with nothing changed: a NULL region, a region not inside the bounds, or an
 * id past the block table.  A region of volume 0 does nothing.  GPU test: tests/test_gpu_region.py. */
aicb_status aicb_scene_update_region(aicb_scene *, const aicb_aab *region, const uint16_t *block_ids_or_null,
                                     uint16_t uniform_id, const uint8_t (*light_or_null)[4]);
/* SpaceChange::BlockEvaluation / BlockIndex (space.rs:1062-1100; updating.rs:128-150): new definitions for EXISTING
 * block indices (an index beyond the table is rejected: aicb_scene_append_blocks adds new ones).  Voxel data is appended to the device pools, and the
 * replaced definitions' voxel data is reclaimed: once a pool's replaced part exceeds its live part, the call compacts
 * that pool on the device (after the wait below, since a frame's hit records hold absolute pool positions).  A pool
 * thus holds at most twice its live data, and aicb_scene_device_bytes counts live and not yet compacted data alike.
 * The 2^32-voxel limit of the brick pool applies to live data.  Cubes
 * holding a block whose classification (invisible / single voxel / voxel brick) changed are re-encoded.  Light is not
 * touched: call aicb_light_relight_blocks with the same indices afterwards to bring the light up to date.  The call first waits for the context's frame in flight and the work queued
 * on the context's stream, and returns once its own device writes are done; it does not wait for other contexts, or
 * for other work on the caller's streams.  GPU test: tests/test_gpu_parity.py::test_block_definition_update_equals_fresh_snapshot. */
aicb_status aicb_scene_update_blocks(aicb_scene *, const uint16_t *indices, const aicb_block_desc *descs, size_t n);
/* SpaceChange::BlockIndex for indices past the table (palette.rs:207-210; UpdatingSpaceRaytracer::update appends them,
 * updating.rs:145-151): the blocks become indices [count, count + n) of the scene's table, where count is the table's
 * size before the call.  From then on they are valid everywhere a block id is: aicb_scene_update_cubes,
 * aicb_scene_update_blocks, aicb_light_edit_and_propagate.  Every output is what a scene created with the longer table
 * gives.  The copies are queued on the context's stream, ordered like aicb_scene_update_cubes (a frame issued later on
 * another stream waits for them); a frame in flight is not disturbed.  The device tables grow geometrically; a table
 * that grows past 16384 blocks re-encodes the cells from 16 to 32 bits on the device.  AICB_ERR_INVALID: NULL with
 * n > 0, count + n > 65536, or a descriptor that scene creation rejects; a rejected call changes nothing.  n == 0 does
 * nothing.  GPU test: tests/test_gpu_append_blocks.py. */
aicb_status aicb_scene_append_blocks(aicb_scene *, const aicb_block_desc *descs, size_t n);
/* SpaceChange::EveryBlock: Mutation::fill_uniform over the whole bounds (space.rs:1461-1474).  The block table becomes
 * exactly [block] and every cube holds id 0; device buffers larger than a new one-block scene needs are freed, and a
 * scene with 32-bit cells goes back to 16-bit cells.  The cells are written on the device.  Light is not touched: the
 * volume, the queue and the set of changed cubes stay as they are, as the reference leaves them; a lit scene's host
 * follows with aicb_light_queue_region(scene, &bounds, 210) and, when it wants the light to move, aicb_light_evaluate.
 * Afterwards every output, and aicb_scene_device_bytes, is what a scene created from the filled Space with
 * aicb_light_download's light gives.  Waiting and ordering are aicb_scene_update_blocks': a frame issued earlier on a
 * caller's stream is the old scene's frame.  AICB_ERR_INVALID: a NULL argument or a descriptor that aicb_scene_create
 * rejects; a rejected call changes nothing.  GPU test: tests/test_gpu_fill_uniform.py. */
aicb_status aicb_scene_fill_uniform(aicb_scene *, const aicb_block_desc *block);
/* Whole light volume replaced (after light propagation on the host or on another rank). */
aicb_status aicb_scene_upload_light(aicb_scene *, const uint8_t (*light)[4], size_t n_texels);
void aicb_scene_destroy(aicb_scene *);
uint64_t aicb_scene_device_bytes(const aicb_scene *);
/* SpaceChange::Physics: Space::set_physics (space.rs:609-630) and, on the light side,
 * LightStorage::maybe_reinitialize_for_physics_change (space/light/updater.rs:80-113).  `sky` is read as
 * aicb_scene_desc::sky is (kind != 0 is Octants); `light_max_distance` means what aicb_scene_desc's does: 0 = None.
 *   - Same sky and same distance: nothing happens (the reference sends no SpaceChange::Physics).
 *   - A new sky: frames use it from then on (Sky::sample, the fog blend, BlockSky::light_outside beyond the bounds) and
 *     so do later light calls.  The light volume, the queue and the set of changed cubes are left as they are, as the
 *     reference leaves them; a host that wants the new sky's light calls aicb_light_fast_evaluate + aicb_light_evaluate.
 *   - Another distance d > 0 (from None or from another d): the light is reinitialised.  The volume is allocated if the
 *     scene has none, fast_evaluate_light runs with the new sky (every texel and every queue entry is written), and every
 *     cube enters the set of changed cubes.  Later light calls use the new maximum_distance.
 *   - None: the light volume and the light state are freed (aicb_scene_device_bytes drops by them), frames read
 *     PackedLight::ONE, the set of changed cubes goes with the state, and light calls are AICB_ERR_INVALID.
 * Afterwards every output equals that of a scene created with the same cells and block table, the new sky, the new
 * light_max_distance and the volume aicb_light_download returns as its light (NULL under None).  The call first waits
 * for the context's frame in flight and the work queued on its stream.  AICB_ERR_INVALID: a NULL scene or sky.
 * AICB_ERR_OOM: the volume or the state could not be allocated.  A failed call changes nothing.
 * GPU test: tests/test_gpu_physics.py. */
aicb_status aicb_scene_set_physics(aicb_scene *, const aicb_sky *sky, uint8_t light_max_distance);

/* ---------------------------------------------------------------------------------------------
 * A scene fed from device memory: the update, light-edit and download calls with their arrays in CUDA buffers of the
 * scene's device (device 0 on a group), for a host whose world changes on the GPU.  Each call leaves the scene, its
 * light, queue and set of changed cubes byte for byte as its host twin does with the same data, with the same errors
 * and messages.
 *   - Pointers: each array is device memory of the scene's device, aligned to its element (4 bytes for cubes and
 *     texels, 2 for ids), checked with cudaPointerGetAttributes before anything is issued: host memory, another
 *     device's memory or a misaligned pointer is AICB_ERR_INVALID.
 *   - Stream: `stream` is a cudaStream_t of the scene's device, or NULL for the context's stream.  The call's kernels
 *     run after the work queued on it before the call (ids a producer kernel wrote there are read correctly), and work
 *     queued on it afterwards runs after the call has read its inputs and written its outputs.  Frames issued later on
 *     any stream see the update, as they see host updates.
 *   - Validation stays on the device: the checks of the host twin (cube in bounds, id < the table's size, region
 *     inside the bounds, LightPhysics::None for the light calls) are reduced by a kernel to a verdict of a few bytes,
 *     the only thing read back before the call decides.  So the calls with ids synchronise with the stream up to their
 *     validation; then they issue their writes, or return AICB_ERR_INVALID with nothing changed.
 *   - Duplicates: a list is sorted stably by cube on the device (CUB radix sort), so update_cubes keeps the last entry
 *     for a cube and light_edit_cubes counts and applies exactly the entries the host loop finds changing.
 *   - The host mirror of the block ids (which aicb_light_edit_cubes, aicb_light_edit_region, aicb_scene_update_blocks
 *     and the host updates use) is not copied back per call: a device update marks it stale, and the first host call
 *     that needs it rebuilds it from the cells with one device-to-host copy of 2 bytes per cube (33.5 MB at 256^3).
 *     aicb_scene_fill_uniform resets it.
 *   - Groups: inputs and outputs are device 0's memory; every replica reads them over peer access or takes a peer copy
 *     of device 0's staged list, and ends identical to the others.  The group calls return once every replica's writes
 *     are done, as the group calls do.
 * The single-context update calls return once their writes are issued; the light edits once their writes are done.
 * GPU test: tests/test_gpu_device_inputs.py. */
/* aicb_scene_update_cubes: int32[n][3] cubes, u16[n] ids, u8[n][4] light or NULL.  n == 0 does nothing. */
aicb_status aicb_scene_update_cubes_device(aicb_scene *, const int32_t (*d_cubes)[3], const uint16_t *d_ids,
                                           const uint8_t (*d_light_or_null)[4], size_t n, void *stream);
/* aicb_scene_update_region: ids Z-major within `region` (NULL: uniform_id), light Z-major within it or NULL.  Every
 * replica's kernels read the arrays where they are.  A uniform fill without light reads nothing and does not wait. */
aicb_status aicb_scene_update_region_device(aicb_scene *, const aicb_aab *region, const uint16_t *d_ids_or_null,
                                            uint16_t uniform_id, const uint8_t (*d_light_or_null)[4], void *stream);
/* aicb_scene_upload_light: one device-to-device copy per replica; nothing to validate on the device, so it does not
 * synchronise. */
aicb_status aicb_scene_upload_light_device(aicb_scene *, const uint8_t (*d_light)[4], size_t n_texels, void *stream);
/* Each cube's block id, Z-major (aicb_scene_desc::block_ids' order), decoded on the device from its cell word (16- or
 * 32-bit cells) into u16[volume] at d_out.  n must be the volume.  Ordered behind the updates queued on the context;
 * does not synchronise on one context. */
aicb_status aicb_scene_download_ids_device(aicb_scene *, uint16_t *d_out, size_t n, void *stream);
/* aicb_light_edit_cubes: the list as above; *n_changed_or_null the changing entries.  Returns once its writes are
 * done. */
aicb_status aicb_light_edit_cubes_device(aicb_scene *, const int32_t (*d_cubes)[3], const uint16_t *d_ids, size_t n,
                                         size_t *n_changed_or_null, void *stream);
/* aicb_light_edit_region: ids Z-major within `region` or NULL for uniform_id.  Returns once its writes are done. */
aicb_status aicb_light_edit_region_device(aicb_scene *, const aicb_aab *region, const uint16_t *d_ids_or_null,
                                          uint16_t uniform_id, size_t *n_changed_or_null, void *stream);
/* aicb_light_download into u8[volume][4] at d_out: a device-to-device copy; does not synchronise on one context. */
aicb_status aicb_light_download_device(aicb_scene *, uint8_t (*d_out)[4], size_t n_texels, void *stream);
/* aicb_scene_update_blocks and aicb_scene_append_blocks with each descriptor's `indices` (u16, Z-major, 2-byte aligned)
 * and `palette` (4-byte aligned) in the scene's device memory; `indices`, the descriptor array and every scalar field
 * stay on the host.  The scene ends as the host twin leaves it with the same data: frames, aicb_scene_device_bytes,
 * light records, cells, compaction, widening.  The host checks what the scalars decide; a kernel checks every voxel
 * index and reads each single voxel's kind, and those bytes are all that is read back before anything is placed
 * (with AICB_BLOCKS_DERIVE_LIGHT, derive's error words are read back after them).  The
 * status and message are the host twin's first; a rejected call changes nothing.  The voxel data is written into the
 * pools on the device, and the cubes of a block whose kind changes are re-encoded on the device, without the host
 * mirror of the block ids.  Ordering is the device calls'; an update also waits for the frame in flight, as
 * aicb_scene_update_blocks does, and both return once their writes are done.  Light is not touched.
 * flags: AICB_BLOCKS_DERIVE_LIGHT ignores the descriptors' light_face_colors, light_color, light_emission and
 * light_opaque_faces and takes them from aicb_derive_block_light's kernels run on the same buffers; light_visible becomes
 * Derived::visible OR the descriptor's light_visible (an animation hint).  A NaN or negative sum fails as
 * aicb_derive_block_light does, naming the block, and changes nothing.  GPU test: tests/test_gpu_device_blocks.py. */
#define AICB_BLOCKS_DERIVE_LIGHT 1u
aicb_status aicb_scene_update_blocks_device(aicb_scene *, const uint16_t *indices, const aicb_block_desc *descs,
                                            size_t n, uint32_t flags, void *stream);
aicb_status aicb_scene_append_blocks_device(aicb_scene *, const aicb_block_desc *descs, size_t n, uint32_t flags,
                                            void *stream);
/* aicb_scene_create with the Space in device memory of the context's device: block_ids (u16, Z-major, 2-byte aligned),
 * light (4-byte aligned, or NULL) and each descriptor's indices and palette, as for aicb_scene_append_blocks_device.
 * The aicb_scene_desc itself, the blocks array, its scalar fields, sky and light_max_distance stay on the host.  The
 * new scene is byte for byte the one aicb_scene_create builds from the same data (cells, block table, light,
 * aicb_scene_device_bytes), and a rejected call fails with aicb_scene_create's status and message, leaves *out NULL
 * and frees what it allocated.  Pointers are checked first; then the bounds, the NULLs and the definitions in
 * aicb_scene_create's order, and "block id out of range" last.  One readback decides: a kernel checks every voxel
 * index and every block id and reads each single voxel's kind.  The cells are encoded on the device from the table's
 * records, and the light is a device-to-device copy.  The scene's host mirror of the block ids starts stale, as
 * after a device update.  flags: AICB_BLOCKS_DERIVE_LIGHT, as for the block calls.  Ordering is the device calls';
 * the call returns once the scene is complete, so the caller may then reuse its buffers.
 * GPU test: tests/test_gpu_device_create.py. */
aicb_status aicb_scene_create_device(aicb_ctx *, const aicb_scene_desc *, uint32_t flags, void *stream,
                                     aicb_scene **out);
/* aicb_scene_fill_uniform with the block's indices and palette in the scene's device memory, checked and placed as
 * aicb_scene_append_blocks_device checks and places them; flags as there.  The scene ends as the host twin leaves it,
 * its host mirror of the block ids reset; a rejected call changes nothing.  Returns once its writes are done. */
aicb_status aicb_scene_fill_uniform_device(aicb_scene *, const aicb_block_desc *block, uint32_t flags, void *stream);

/* ---------------------------------------------------------------------------------------------
 * draw(): replaces RtRenderer::draw_rgba / RtRenderer::draw::<ColorBuf> and the Rayon pixel
 * dispatch trace_scene_to_image_impl (renderer.rs:183-220, 282-308, 516-556).
 * Host-buffer variants copy device->host inside the call (blocking, like draw_rgba).
 * `out_len` must equal aicb_shard_pixel_count(camera, shard) or AICB_ERR_INVALID is returned.
 * Pixels of the shard's rows are packed in increasing row order, row-major, top-left origin.
 * ------------------------------------------------------------------------------------------- */
size_t aicb_shard_pixel_count(const aicb_camera *, const aicb_shard *shard_or_null);

/* == draw_rgba: sRGB8 RGBA, post_process_color + to_srgb8 applied (renderer.rs:287-291). */
aicb_status aicb_render_srgb8(aicb_scene *, const aicb_camera *, const aicb_options *,
                              const aicb_shard *shard_or_null,
                              uint8_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);

/* == the per-pixel colour of raytrace_to_texture (all-is-cubes-gpu/src/raytrace_to_texture.rs:645-661):
 * ColorBuf::into_premultiplied_rgba (all-is-cubes/src/raytracer_components.rs:70-77) with the camera's exposure
 * applied to r, g, b, rounded to IEEE binary16 like half::f16::from_f32; not tone-mapped (the caller's GPU
 * postprocessing does that).  out[i] = {r, g, b, a} as raw f16 bits. */
aicb_status aicb_render_rgba16f(aicb_scene *, const aicb_camera *, const aicb_options *,
                                const aicb_shard *shard_or_null,
                                uint16_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);

/* == draw::<ColorBuf> (+ DepthBuf, + Position): raw accumulators for parity and other callers.
 * out_colorbuf: light.xyz, transmittance (raytracer_components.rs:20-39).
 * depth_or_null: DepthBuf::depth (accum.rs:254-311) of the first Hit carrying a t_distance.
 * hit_or_null: Position of the first surface hit. */
aicb_status aicb_render_colorbuf(aicb_scene *, const aicb_camera *, const aicb_options *,
                                 const aicb_shard *shard_or_null,
                                 float (*out_colorbuf)[4], double *depth_or_null, aicb_hit *hit_or_null,
                                 uint32_t *steps_or_null, size_t out_len, aicb_render_info *info_or_null);

/* == print_space's image (raytracer/text.rs:139-180): per pixel the CharacterBuf state (text.rs:52-123) — the block
 * index of the first block the ray hit, or one of AICB_TEXT_*.  The caller prints each value with the string its block
 * data gives that block (D::from_block). */
aicb_status aicb_render_text(aicb_scene *, const aicb_camera *, const aicb_options *, int32_t *out, size_t out_len,
                             aicb_render_info *info_or_null);

/* == RtScene::trace_ray_through_layers + draw_rgba (renderer.rs:454-478, 282-308): the UI layer (its own Space and
 * camera, traced without sky), the backdrop colour (StandardCameras' UiViewState::backdrop; NULL or transparent = none),
 * then the world layer continuing in the same accumulator; a pixel that is still not opaque (no world layer) is
 * painted `no_world_rgba` (palette::NO_WORLD_TO_SHOW, linear RGBA; NULL = leave).  Either layer may be NULL.  Both
 * scenes must belong to one context and both cameras to one framebuffer size; the world layer's options choose the
 * antialiasing sample points and the post-processing.  The info text of draw(info_text) is drawn by the caller over
 * the returned image (renderer.rs:659-683 needs the font of the universe). */
typedef struct aicb_layer {
    aicb_scene *scene;
    const aicb_camera *camera;
    const aicb_options *options;
} aicb_layer;
aicb_status aicb_render_layers_srgb8(const aicb_layer *world_or_null, const aicb_layer *ui_or_null,
                                     const float backdrop_rgba[4], const float no_world_rgba[4],
                                     uint8_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);

/* == RaytraceToTexture::do_some_tracing's trace_one for a batch (all-is-cubes-gpu/src/raytrace_to_texture.rs:591-683):
 * the layers traced as aicb_render_layers_srgb8 traces them, into the Split accumulator (:922-977), stored as the two
 * texels of a pixel.
 *   out_rgba16f: ColorBuf::into_premultiplied_rgba with r, g, b scaled by the exposure (aicb_camera::exposure) of the
 *                layer the pixel belongs to (1 for neither), as raw IEEE binary16 bits (half::f16::from_f32).
 *   out_depth:   DepthBuf::depth().clamp(0, 1) through depth_transform (euclid's transform_point3d_homogeneous of
 *                (0, 0, d), z / w in f64), as f32, times +1 for the world layer and -1 for the UI layer or neither.
 * A pixel belongs to the layer of its first hit after which the accumulator is not fully transparent; the backdrop
 * belongs to the UI layer and NO_WORLD_TO_SHOW to the world.  With antialiasing the four samples are reduced by
 * Split::mean: ColorBuf mean, least depth, the first sample's layer that has one.
 * depth_transform: m11..m44 (row-vector convention), as the caller builds it from the world camera
 * (projection_matrix().pre_translate((0, 0, -near)).pre_scale(0, 0, -(view_distance - near)), :613-618).
 * pixels_or_null: linear framebuffer indices y * fb_width + x, any order, repeats allowed; outputs are packed in list
 * order.  With NULL, n_pixels must be fb_width * fb_height and the outputs are the whole texture, row-major.
 * n_pixels == 0 does nothing.  AICB_ERR_INVALID: an index >= fb_width * fb_height, a length mismatch, or what
 * aicb_render_layers_srgb8 rejects.  The lead layer's antialiasing option chooses the sample points. */
aicb_status aicb_render_layers_texture(const aicb_layer *world_or_null, const aicb_layer *ui_or_null,
                                       const float backdrop_rgba[4], const float no_world_rgba[4],
                                       const double depth_transform[16],
                                       const uint32_t *pixels_or_null, size_t n_pixels,
                                       uint16_t (*out_rgba16f)[4], float *out_depth,
                                       aicb_render_info *info_or_null);

/* == the desktop app's terminal frame (all-is-cubes-desktop/src/terminal.rs:114-142): RtRenderer<CharacterRtData>::draw
 * into ColorCharacterBuf (:341-394) and ColorCharacterBuf::output (:355-366) per pixel, the layers traced as
 * aicb_render_layers_srgb8 traces them.  The accumulator stops where that call's does (its ColorBuf's opacity), so the
 * hits, step counts and cubes_traced are that call's; CharacterBuf (raytracer/text.rs:52-123) follows every hit the
 * colour gets: the first surface names its block, Exception::Incomplete before one is "X", the backdrop, debug_pixel_cost
 * and NO_WORLD_TO_SHOW (which replaces the whole accumulator) are " " (AICB_TEXT_BLANK), and a ray that counted a step
 * entered the space.  The four antialiasing samples are reduced by ColorBuf::mean and CharacterBuf::mean (the first
 * sample with a hit gives the text; EnteredSpace only if every sample entered).
 *   rgba:  Camera::post_process_color(Rgba::from(ColorBuf)) of the world layer's camera and options (the UI layer's
 *          without a world): exposure, then tone mapping, linear f32, the value aicb_render_layers_srgb8 encodes.
 *   text:  the block index (>= 0) the caller maps with CharacterRtData::from_block, or AICB_TEXT_*.
 *   layer: the layer whose Space the block index belongs to (AICB_LAYER_WORLD / _UI); AICB_LAYER_NONE for text < 0.
 * Arguments, validation and options are aicb_render_layers_srgb8's; out_len pixels, row-major. */
enum { AICB_LAYER_NONE = 0, AICB_LAYER_WORLD = 1, AICB_LAYER_UI = 2 };
typedef struct aicb_terminal_pixel {
    float rgba[4];
    int32_t text;
    int32_t layer;
} aicb_terminal_pixel;
aicb_status aicb_render_layers_terminal(const aicb_layer *world_or_null, const aicb_layer *ui_or_null,
                                        const float backdrop_rgba[4], const float no_world_rgba[4],
                                        aicb_terminal_pixel *out, size_t out_len, aicb_render_info *info_or_null);

/* == render_orthographic (raytracer/ortho.rs:30-84): the five axis-aligned views of MultiOrthoCamera (:143-199) in one
 * image at `resolution` pixels per cube (the reference uses 32), UNALTERED_COLORS, sRGB8 without post-processing,
 * transparent between the views.  aicb_ortho_image_size gives the image size for a scene. */
aicb_status aicb_ortho_image_size(const aicb_scene *, uint32_t resolution, uint32_t *width, uint32_t *height);
aicb_status aicb_render_orthographic(aicb_scene *, uint32_t resolution, uint8_t (*out)[4], size_t out_len,
                                     aicb_render_info *info_or_null);

/* Device-resident output (for multi-GPU gather and kernel-only timing): `d_out` is a device
 * pointer on the ctx's device with room for out_len pixels; `stream` is a cudaStream_t (0 =
 * the ctx stream). Does not synchronise; info (if given) is filled by
 * aicb_render_finish(). */
aicb_status aicb_render_srgb8_device(aicb_scene *, const aicb_camera *, const aicb_options *,
                                     const aicb_shard *shard_or_null,
                                     void *d_out, size_t out_len, void *stream);
/* As above, but `d_frame` is a FULL framebuffer (fb_width*fb_height pixels) and the shard's pixels
 * are stored at their framebuffer positions.  `d_frame` may be peer memory of another GPU mapped
 * into this process (cudaIpcOpenMemHandle / P2P): the trace kernel's epilogue then delivers its
 * row strips straight into the root GPU's frame over NVLink, replacing the gather collective. */
aicb_status aicb_render_srgb8_device_frame(aicb_scene *, const aicb_camera *, const aicb_options *,
                                           const aicb_shard *shard_or_null,
                                           void *d_frame, size_t frame_len, void *stream);
aicb_status aicb_render_finish(aicb_scene *, aicb_render_info *info_or_null);

/* Every output in the caller's device memory: the outputs of a call are stored where these pointers say, by the
 * kernels that compute them, and nothing is copied to the host.  Each pointer is NULL or device memory of the call's
 * device (the scene's; device 0 on a group), checked with cudaPointerGetAttributes before anything is issued: host
 * memory or another device's memory is AICB_ERR_INVALID.  Element types and layouts are the host calls':
 *   world frames and ray batches: srgb8, rgba16f, colorbuf + depth + hit + steps, text;
 *   layered frames: srgb8, terminal; texture targets: texel_rgba16f + texel_depth.
 * A call accepts the outputs of one host call, and only those: {srgb8}, {rgba16f}, a non-empty subset of
 * {colorbuf, depth, hit, steps} (the group calls need colorbuf, as aicb_group_render_colorbuf does), {text}; layered:
 * {srgb8}, {terminal}, {texel_rgba16f and texel_depth}.  Any other combination, or a pointer the call cannot fill, is
 * AICB_ERR_INVALID.  `len` is the host call's out_len (pixels, rays or listed pixels).  `full_frame` (aicb_render_device
 * only, 0 elsewhere) has aicb_render_srgb8_device_frame's meaning: len = fb_width * fb_height and the shard's pixels are
 * stored at their framebuffer positions. */
typedef struct aicb_device_outputs {
    uint8_t (*srgb8)[4];
    uint16_t (*rgba16f)[4];
    float (*colorbuf)[4];
    double *depth;
    aicb_hit *hit;
    uint32_t *steps;
    int32_t *text;
    uint16_t (*texel_rgba16f)[4];
    float *texel_depth;
    aicb_terminal_pixel *terminal;
    size_t len;
    uint32_t full_frame;
    uint32_t _pad;
} aicb_device_outputs;

/* Asynchronous calls on one context, issued on `stream` (a cudaStream_t of the scene's device; NULL = the context's
 * stream), which nothing synchronises: aicb_render_finish on the scene completes the call (for a layered call, the
 * world layer's scene, or the UI layer's without a world), fills info and returns AICB_ERR_RETRY after a hit-stream
 * overflow, after which the caller issues the same call again.  The outputs are final once the stream has passed the
 * call's work; the inputs (rays, pixel list) must stay valid until then.  A frame on a caller's stream waits for the
 * context's previous frame and for the scene updates queued before it; the scene must not change again before the
 * frame is finished.  A context tracks one frame: any render call on it (another asynchronous call, a host call, on
 * any of its scenes) starts a new frame whose counters and overflow flag replace this one's, so aicb_render_finish
 * would report that frame and could miss this one's overflow.  Finish each asynchronous call before the context's next
 * render call.  Outputs, info and validation are those of the host calls, bit for bit.  Every pointer must be aligned
 * to its elements' stores (16 bytes for colorbuf; 8 for rgba16f, depth, texel_rgba16f, terminal and the ray batch; 4
 * for the others), AICB_ERR_INVALID otherwise.
 *   aicb_render_device: the world-only frames of aicb_render_srgb8 / _rgba16f / _colorbuf / _text.
 *   aicb_trace_rays_device: aicb_trace_rays with the batch read from device memory of the scene's device.
 *   aicb_render_layers_device: aicb_render_layers_srgb8 (outs->srgb8), _terminal (outs->terminal) or _texture
 *     (outs->texel_rgba16f and texel_depth, with depth_transform and the pixel list; n_pixels is 0 otherwise).  The UI
 *     pass and the world pass are issued back to back; an overflow in either surfaces as AICB_ERR_RETRY.  The pixel list
 *     is device memory of the scene's device and is read as it is: unlike the host call's, its indices are not checked
 *     (an index >= fb_width * fb_height traces a ray outside the viewport into its own list position). */
aicb_status aicb_render_device(aicb_scene *, const aicb_camera *, const aicb_options *, const aicb_shard *shard_or_null,
                               const aicb_device_outputs *outs, void *stream);
aicb_status aicb_trace_rays_device(aicb_scene *, const double (*d_origin_dir)[6], size_t n, const aicb_options *,
                                   const aicb_device_outputs *outs, void *stream);
aicb_status aicb_render_layers_device(const aicb_layer *world_or_null, const aicb_layer *ui_or_null,
                                      const float backdrop_rgba[4], const float no_world_rgba[4],
                                      const double depth_transform_or_null[16], const uint32_t *d_pixels_or_null,
                                      size_t n_pixels, const aicb_device_outputs *outs, void *stream);

/* A batch of views of one scene drawn as one frame: n_views cameras (a world for many characters, sensors, split
 * screens), each view RtRenderer::draw for its camera, bit for bit the single-camera call's output.  The host forms take
 * the arguments and give the outputs of aicb_render_srgb8 / _rgba16f / _colorbuf / _text, with the camera table and
 * n_views in place of the one camera, and no shard:
 *   - outputs are view-major: view v's pixel (x, y) is element v * W * H + y * W + x, and out_len must be
 *     n_views * W * H;
 *   - each view uses its own camera's inverse_projection_view and exposure; everything in aicb_options is shared;
 *   - every camera must have the same fb_width x fb_height (W x H), AICB_ERR_INVALID otherwise;
 *   - info covers the batch: cubes_traced, rays and counters are the sums of the single calls', flaws are ORed, and
 *     kernel_ms is the batch's time;
 *   - n_views == 0 or W * H == 0 does nothing;
 *   - AICB_ERR_INVALID also for NULL cameras with n_views > 0, and for a batch whose task count
 *     (n_views * ceil(W / 8) * ceil(H / 4) * 32 * samples, 4 samples with antialiasing) reaches 2^32.
 * Every argument is checked before anything is issued: a rejected call writes nothing.  The calls block, and re-issue
 * the batch after a hit-stream overflow as the single-camera host calls do. */
aicb_status aicb_render_views_srgb8(aicb_scene *, const aicb_camera *cameras, size_t n_views, const aicb_options *,
                                    uint8_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_render_views_rgba16f(aicb_scene *, const aicb_camera *cameras, size_t n_views, const aicb_options *,
                                      uint16_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_render_views_colorbuf(aicb_scene *, const aicb_camera *cameras, size_t n_views, const aicb_options *,
                                       float (*out_colorbuf)[4], double *depth_or_null, aicb_hit *hit_or_null,
                                       uint32_t *steps_or_null, size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_render_views_text(aicb_scene *, const aicb_camera *cameras, size_t n_views, const aicb_options *,
                                   int32_t *out, size_t out_len, aicb_render_info *info_or_null);
/* The batch with the camera table (8-byte aligned) and the outputs in device memory of the scene's device.  The
 * framebuffer size is the call's: only inverse_projection_view and exposure are read from each camera, whose own size
 * fields are not checked.  The outputs are the world-frame sets aicb_render_device accepts, with full_frame 0 and len
 * n_views * fb_width * fb_height.  Otherwise aicb_render_device's contract: issued on `stream`, completed by
 * aicb_render_finish, AICB_ERR_RETRY after an overflow. */
aicb_status aicb_render_views_device(aicb_scene *, const aicb_camera *d_cameras, size_t n_views, uint32_t fb_width,
                                     uint32_t fb_height, const aicb_options *, const aicb_device_outputs *outs,
                                     void *stream);

/* Full-frame buffers shared between the ranks of one node (one process per GPU): the root creates
 * the frame on its GPU and publishes a 64-byte CUDA IPC handle; the other ranks open it on THEIR
 * device (peer access over NVLink is enabled lazily) and pass the mapped pointer to
 * aicb_render_srgb8_device_frame().  aicb_frame_read() is the root's device->host copy. */
aicb_status aicb_frame_create(aicb_ctx *, size_t n_pixels, void **d_frame, uint8_t handle_out[64]);
aicb_status aicb_frame_open(aicb_ctx *, const uint8_t handle[64], void **d_frame);
aicb_status aicb_frame_close(aicb_ctx *, void *d_frame, int opened);
aicb_status aicb_frame_read(aicb_ctx *, const void *d_frame, uint8_t (*out)[4], size_t n_pixels, void *stream);
/* Delivery without a collective.  A shared frame carries two monotonic counters behind its pixels:
 *   aicb_frame_signal          (every rank, after aicb_render_srgb8_device_frame on the same stream): "my strips of this
 *                              frame are stored" — arrived += 1, system-scope fence first so the pixels are visible;
 *   aicb_frame_wait_arrived    (owner): stream-ordered wait until arrived >= count (= ranks x frames so far);
 *   aicb_frame_release         (owner): consumed := frame_id once it is through with the frame (copied, displayed);
 *   aicb_frame_wait_consumed   (every rank, before storing into the frame again): wait until consumed >= frame_id.
 * All four are stream operations (one-thread kernels), none touches the host.  A wait gives up after ~2 s;
 * aicb_frame_timed_out reports it.  `n_pixels` is the frame's pixel count as given to aicb_frame_create. */
aicb_status aicb_frame_signal(aicb_ctx *, void *d_frame, size_t n_pixels, void *stream);
aicb_status aicb_frame_wait_arrived(aicb_ctx *, void *d_frame, size_t n_pixels, uint32_t count, void *stream);
aicb_status aicb_frame_release(aicb_ctx *, void *d_frame, size_t n_pixels, uint32_t frame_id, void *stream);
aicb_status aicb_frame_wait_consumed(aicb_ctx *, void *d_frame, size_t n_pixels, uint32_t frame_id, void *stream);
aicb_status aicb_frame_timed_out(aicb_ctx *, void *d_frame, size_t n_pixels, uint32_t *out);

/* ---------------------------------------------------------------------------------------------
 * Several GPUs from ONE process (csrc/group.cu): replaces the Rayon rows x pixels dispatch of
 * trace_scene_to_image_impl (renderer.rs:516-556) across devices for hosts that own their process (the Rust
 * `impl HeadlessRenderer`, INTEGRATION.md).  The scene is replicated on every device of the group; a frame is cut into
 * interleaved 16-row strips (strip s -> device s mod n); every device's last kernel stores its pixels straight into
 * device 0's frame over NVLink (peer access) and device 0 copies the frame to the caller once the other devices'
 * completion events have fired: no collective, no host thread per GPU.  The same device may be named more than once
 * (tests).  aicb_render_info: counters summed over the devices, times = the slowest device's.
 * ------------------------------------------------------------------------------------------- */
typedef struct aicb_group aicb_group;
typedef struct aicb_group_scene aicb_group_scene;
aicb_status aicb_group_create(const int *device_ids, int n_devices, aicb_group **out);
void aicb_group_destroy(aicb_group *);
int aicb_group_size(const aicb_group *);
aicb_status aicb_group_scene_create(aicb_group *, const aicb_scene_desc *, aicb_group_scene **out);
void aicb_group_scene_destroy(aicb_group_scene *);
aicb_status aicb_group_scene_update_cubes(aicb_group_scene *, const int32_t (*cubes)[3], const uint16_t *block_ids,
                                          const uint8_t (*light)[4], size_t n);
/* aicb_scene_update_region on every replica, holding every context of the group: validated against replica 0, then
 * every replica stages the arrays in its own context and writes its own cells and texels. */
aicb_status aicb_group_scene_update_region(aicb_group_scene *, const aicb_aab *region, const uint16_t *block_ids_or_null,
                                           uint16_t uniform_id, const uint8_t (*light_or_null)[4]);
/* == draw_rgba on the whole group: out_len must be fb_width * fb_height; the options apply as given (include_sky too).
 * The frame is issued on every device before any is waited for; a device whose hit stream overflowed is re-issued
 * alone.  The call holds every context of the group until it returns. */
aicb_status aicb_group_render_srgb8(aicb_group_scene *, const aicb_camera *, const aicb_options *,
                                    uint8_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);
/* aicb_scene_update_blocks (SpaceChange::BlockEvaluation / BlockIndex, updating.rs:128-150) and aicb_scene_upload_light
 * on every replica.  These calls and aicb_group_scene_update_cubes hold every context of the group until they return.
 * The update is validated against replica 0 first: a rejected call changes no replica.  Whether a
 * pool is compacted is decided from replica 0's table, and every replica compacts, so the tables stay identical.  The
 * update does not touch light: aicb_group_light_relight_blocks follows it.  A call that fails after validation, for want
 * of device memory on a replica other than the first (placing the definitions, or compacting a pool, there or in
 * aicb_group_scene_append_blocks), may leave the replicas' tables different: destroy the group scene and create it
 * again. */
aicb_status aicb_group_scene_update_blocks(aicb_group_scene *, const uint16_t *indices, const aicb_block_desc *descs,
                                           size_t n);
aicb_status aicb_group_scene_upload_light(aicb_group_scene *, const uint8_t (*light)[4], size_t n_texels);
/* aicb_scene_set_physics on every replica, holding every context of the group.  It is decided against replica 0 before
 * any replica changes, and every replica takes the sky.  A reinitialisation runs as aicb_group_light_fast_evaluate does
 * (device 0 computes, the others take peer copies; the set of changed cubes and the queue are device 0's), so the
 * replicas stay identical.  A failed call changes no replica. */
aicb_status aicb_group_scene_set_physics(aicb_group_scene *, const aicb_sky *sky, uint8_t light_max_distance);
/* aicb_scene_append_blocks on every replica, validated against replica 0 before any replica changes: a rejected call
 * changes no replica.  The call holds every context of the group; a table that grows past 16384 blocks widens every
 * replica's cells on its own device. */
aicb_status aicb_group_scene_append_blocks(aicb_group_scene *, const aicb_block_desc *descs, size_t n);
/* aicb_scene_fill_uniform on every replica, holding every context of the group: the block is validated and flattened
 * once, so a rejected call changes no replica, then every replica is filled on its own device. */
aicb_status aicb_group_scene_fill_uniform(aicb_group_scene *, const aicb_block_desc *block);
/* The device-input calls (aicb_scene_update_cubes_device ..) on the group: arrays in device 0's memory, validated on
 * device 0 before any replica changes; every replica ends identical; each call returns once every replica's writes
 * are done (for the downloads, once device 0's output is final).  aicb_group_scene_download_ids_device and
 * aicb_group_light_download_device read replica 0. */
aicb_status aicb_group_scene_update_cubes_device(aicb_group_scene *, const int32_t (*d_cubes)[3], const uint16_t *d_ids,
                                                 const uint8_t (*d_light_or_null)[4], size_t n, void *stream);
aicb_status aicb_group_scene_update_region_device(aicb_group_scene *, const aicb_aab *region,
                                                  const uint16_t *d_ids_or_null, uint16_t uniform_id,
                                                  const uint8_t (*d_light_or_null)[4], void *stream);
aicb_status aicb_group_scene_upload_light_device(aicb_group_scene *, const uint8_t (*d_light)[4], size_t n_texels,
                                                 void *stream);
aicb_status aicb_group_scene_download_ids_device(aicb_group_scene *, uint16_t *d_out, size_t n, void *stream);
aicb_status aicb_group_light_edit_cubes_device(aicb_group_scene *, const int32_t (*d_cubes)[3], const uint16_t *d_ids,
                                               size_t n, size_t *n_changed_or_null, void *stream);
aicb_status aicb_group_light_edit_region_device(aicb_group_scene *, const aicb_aab *region,
                                                const uint16_t *d_ids_or_null, uint16_t uniform_id,
                                                size_t *n_changed_or_null, void *stream);
aicb_status aicb_group_light_download_device(aicb_group_scene *, uint8_t (*d_out)[4], size_t n_texels, void *stream);
/* The block definitions' voxels are device 0's memory, checked once there; every replica's kernels read them over
 * peer access and every replica's table ends identical.  Returns once every replica's writes are done. */
aicb_status aicb_group_scene_update_blocks_device(aicb_group_scene *, const uint16_t *indices,
                                                  const aicb_block_desc *descs, size_t n, uint32_t flags, void *stream);
aicb_status aicb_group_scene_append_blocks_device(aicb_group_scene *, const aicb_block_desc *descs, size_t n,
                                                  uint32_t flags, void *stream);
/* aicb_scene_create_device and aicb_scene_fill_uniform_device on the group: the inputs are device 0's memory, checked
 * once there.  Every replica's table is written by its own kernels, and every replica encodes its own cells from
 * device 0's ids, read over peer access; the light is a peer copy per replica.  Each returns once every replica is
 * complete. */
aicb_status aicb_group_scene_create_device(aicb_group *, const aicb_scene_desc *, uint32_t flags, void *stream,
                                           aicb_group_scene **out);
aicb_status aicb_group_scene_fill_uniform_device(aicb_group_scene *, const aicb_block_desc *block, uint32_t flags,
                                                 void *stream);

/* == RtScene::trace_ray_through_layers + draw_rgba (renderer.rs:454-478, 282-308) and RaytraceToTexture::do_some_tracing's
 * trace_one (all-is-cubes-gpu/src/raytrace_to_texture.rs:591-683) on the whole group: the arguments, the validation and
 * the outputs of aicb_render_layers_srgb8 / aicb_render_layers_texture, bit for bit, with group scenes in place of
 * scenes; both layers must be scenes of the same group (AICB_ERR_INVALID otherwise).  A whole frame or texture is cut
 * into interleaved 16-row strips as aicb_group_render_srgb8 cuts it; a pixel list into contiguous ranges of whole
 * 32-entry warps, one per device (a list of fewer than 32 x devices entries uses fewer devices).  Every device stores
 * its outputs straight into device 0's buffers, in framebuffer or list order.  Each pass (UI, then world) is issued on
 * every device before any device's pass is waited for; a pass whose hit stream overflowed is re-issued on that device
 * alone.  aicb_render_info: counters summed over the devices, times = the slowest device's, its passes summed. */
typedef struct aicb_group_layer {
    aicb_group_scene *scene;
    const aicb_camera *camera;
    const aicb_options *options;
} aicb_group_layer;
aicb_status aicb_group_render_layers_srgb8(const aicb_group_layer *world_or_null, const aicb_group_layer *ui_or_null,
                                           const float backdrop_rgba[4], const float no_world_rgba[4],
                                           uint8_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_group_render_layers_texture(const aicb_group_layer *world_or_null, const aicb_group_layer *ui_or_null,
                                             const float backdrop_rgba[4], const float no_world_rgba[4],
                                             const double depth_transform[16],
                                             const uint32_t *pixels_or_null, size_t n_pixels,
                                             uint16_t (*out_rgba16f)[4], float *out_depth,
                                             aicb_render_info *info_or_null);

/* == aicb_render_layers_terminal on the whole group, bit for bit: its arguments with group scenes (both of the same
 * group), the frame cut into interleaved 16-row strips as aicb_group_render_layers_srgb8 cuts it, every device storing
 * into device 0's buffer. */
aicb_status aicb_group_render_layers_terminal(const aicb_group_layer *world_or_null, const aicb_group_layer *ui_or_null,
                                              const float backdrop_rgba[4], const float no_world_rgba[4],
                                              aicb_terminal_pixel *out, size_t out_len, aicb_render_info *info_or_null);

/* The world-only outputs of one context on the whole group: the arguments, the validation (against replica 0, before
 * any device is touched) and the outputs of aicb_render_colorbuf / _rgba16f / _text / _orthographic /
 * aicb_ortho_image_size and aicb_trace_rays, bit for bit, with a group scene in place of a scene.  Frames are whole
 * frames (out_len = fb_width * fb_height, no shard): each is cut into interleaved 16-row strips as
 * aicb_group_render_srgb8 cuts it.  A ray batch is cut into contiguous ranges of whole 32-ray warps, one per device, as
 * even as whole warps allow (a batch of fewer than 32 x devices rays uses fewer devices); each device uploads only its
 * own range.  The orthographic image's five views are built on the devices and their pixels cut the same way.  Every
 * device stores its outputs straight into device 0's buffers, in framebuffer or batch order, and device 0 copies the
 * outputs the caller asked for (the non-NULL ones) to the caller.  Unlike the single-context calls, out_colorbuf may
 * not be NULL when there are pixels or rays (AICB_ERR_INVALID).  A device whose hit stream overflowed is re-issued
 * alone.  aicb_render_info: counters summed over the devices, times = the slowest device's. */
aicb_status aicb_group_render_colorbuf(aicb_group_scene *, const aicb_camera *, const aicb_options *,
                                       float (*out_colorbuf)[4], double *depth_or_null, aicb_hit *hit_or_null,
                                       uint32_t *steps_or_null, size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_group_render_rgba16f(aicb_group_scene *, const aicb_camera *, const aicb_options *,
                                      uint16_t (*out)[4], size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_group_trace_rays(aicb_group_scene *, const double (*origin_dir)[6], size_t n, const aicb_options *,
                                  float (*out_colorbuf)[4], double *depth_or_null, aicb_hit *hit_or_null,
                                  uint32_t *steps_or_null, aicb_render_info *info_or_null);
aicb_status aicb_group_render_text(aicb_group_scene *, const aicb_camera *, const aicb_options *,
                                   int32_t *out, size_t out_len, aicb_render_info *info_or_null);
aicb_status aicb_group_ortho_image_size(const aicb_group_scene *, uint32_t resolution, uint32_t *width, uint32_t *height);
aicb_status aicb_group_render_orthographic(aicb_group_scene *, uint32_t resolution, uint8_t (*out)[4],
                                           size_t out_len, aicb_render_info *info_or_null);

/* aicb_render_device, aicb_trace_rays_device and aicb_render_layers_device on the whole group: the group calls above
 * with their cuts, validation and outputs, bit for bit, every device storing straight into the caller's device-0
 * buffers (aicb_device_outputs), and no copy to the host.  The ray batch and the pixel list are device-0 memory, which
 * every device reads over peer access.  Unlike the single-context calls these block, as the other group calls do: a
 * device whose hit stream overflowed is re-issued alone, and the call returns once device 0's buffers are final, with
 * info filled.  `stream` (a cudaStream_t of device 0, or NULL): every device's work starts after the work queued on it
 * before the call (which may be writing the inputs), and it waits for the call's completion events, so work queued
 * on it afterwards is ordered behind the outputs without the host.  A fully asynchronous group call is not offered. */
aicb_status aicb_group_render_device(aicb_group_scene *, const aicb_camera *, const aicb_options *,
                                     const aicb_device_outputs *outs, void *stream, aicb_render_info *info_or_null);
aicb_status aicb_group_trace_rays_device(aicb_group_scene *, const double (*d_origin_dir)[6], size_t n,
                                         const aicb_options *, const aicb_device_outputs *outs, void *stream,
                                         aicb_render_info *info_or_null);
aicb_status aicb_group_render_layers_device(const aicb_group_layer *world_or_null, const aicb_group_layer *ui_or_null,
                                            const float backdrop_rgba[4], const float no_world_rgba[4],
                                            const double depth_transform_or_null[16],
                                            const uint32_t *d_pixels_or_null, size_t n_pixels,
                                            const aicb_device_outputs *outs, void *stream,
                                            aicb_render_info *info_or_null);

/* The batches of views (aicb_render_views_*) on the whole group, bit for bit one context's: view v is drawn by device
 * v mod N (views differ in cost, as row strips do), and every device stores its views into device 0's buffers.  The
 * device form blocks and orders `stream` as aicb_group_render_device does; its camera table is device-0 memory, which
 * every device reads over peer access. */
aicb_status aicb_group_render_views_srgb8(aicb_group_scene *, const aicb_camera *cameras, size_t n_views,
                                          const aicb_options *, uint8_t (*out)[4], size_t out_len,
                                          aicb_render_info *info_or_null);
aicb_status aicb_group_render_views_rgba16f(aicb_group_scene *, const aicb_camera *cameras, size_t n_views,
                                            const aicb_options *, uint16_t (*out)[4], size_t out_len,
                                            aicb_render_info *info_or_null);
aicb_status aicb_group_render_views_colorbuf(aicb_group_scene *, const aicb_camera *cameras, size_t n_views,
                                             const aicb_options *, float (*out_colorbuf)[4], double *depth_or_null,
                                             aicb_hit *hit_or_null, uint32_t *steps_or_null, size_t out_len,
                                             aicb_render_info *info_or_null);
aicb_status aicb_group_render_views_text(aicb_group_scene *, const aicb_camera *cameras, size_t n_views,
                                         const aicb_options *, int32_t *out, size_t out_len,
                                         aicb_render_info *info_or_null);
aicb_status aicb_group_render_views_device(aicb_group_scene *, const aicb_camera *d_cameras, size_t n_views,
                                           uint32_t fb_width, uint32_t fb_height, const aicb_options *,
                                           const aicb_device_outputs *outs, void *stream,
                                           aicb_render_info *info_or_null);

/* ---------------------------------------------------------------------------------------------
 * Texture targets: the state RaytraceToTexture::Inner keeps around trace_one (all-is-cubes-gpu/src/raytrace_to_texture.rs),
 * on the device: the update strategy and its position, dirty_pixels, and the colour and depth render targets.  The
 * RtRenderer is not part of it: the layers are passed to each trace, as aicb_render_layers_texture takes them.
 * rays_per_frame and its 2 ms budget rule (:733-744) stay with the caller, which passes the batch size and times the
 * call with its own clock.  Reprojection (UpdateStrategy::want_reprojection) is not offered: the reference never
 * takes it (:140).
 *   create: a w x h render viewport (w, h >= 1 and w * h <= 2^30 - 1; AICB_ERR_INVALID otherwise) with
 *     AICB_TEXTURE_INCREMENTAL (PixelPicker, :835-918: the pixels stably sorted by their Chebyshev distance from the
 *     centre plus a dither, the order built and kept on the device, 4 bytes per pixel) or AICB_TEXTURE_CONSISTENT
 *     (`next`, :704-727; point_from_pixel_index wraps, :912-918).  Both targets hold zero bits (a new DrawableTexture),
 *     the pick position is 0 and dirty_pixels = cycle_length (:188).
 *   cycle_length: Incremental 2 * max(central, w * h - central) with central = min(60000, w * h / 4) (:877-886);
 *     Consistent w * h.
 *   mark_dirty: dirty_pixels = cycle_length (RaytraceToTexture::dirty, :587-589), for a host whose RtRenderer::update
 *     reported a change.
 *   resize (:311-324): the same size does nothing.  Another size makes new targets of zero bits and, for Incremental,
 *     a new order whose pick position is 0 (PixelPicker::new); Consistent keeps its position.  dirty_pixels is left as
 *     it is, as the reference leaves it.  A failed resize changes nothing.
 *   trace (do_some_tracing, :591-745): with dirty_pixels == 0 nothing is traced and *n_traced = 0.  Otherwise picks
 *     p .. p + n - 1 (p the pick position) are traced as aicb_render_layers_texture traces a pixel list, each pick's two
 *     texels are stored at its framebuffer position in the targets (store_one, :685-690; a pixel picked twice in a
 *     batch gets the same bits twice), p += n, dirty_pixels -= min(n, dirty_pixels), and *n_traced = n.  The picks are
 *     computed by the kernel that lists the batch's rays: no pixel list and no texel crosses to or from the host.
 *     AICB_ERR_INVALID: what aicb_render_layers_texture rejects, a camera whose framebuffer size is not the target's,
 *     layers whose scenes are not on the target's context (of the target's group), or n > 2^30 - 1.
 *   state: the size, the strategy, dirty_pixels, the pick position and cycle_length.
 *   picks: the linear indices y * w + x of picks start .. start + n - 1, from the device code that feeds a batch.
 *   buffers: device pointers, on the context's device, to the w * h texels of each target, row-major: the colour texels
 *     as aicb_render_layers_texture's out_rgba16f (4 x f16 bits), the depth texels as its out_depth (f32); valid until
 *     the next resize or destroy.  read: a copy of them (n must be w * h; either pointer may be NULL).
 * Every call is blocking: it holds the target's context locks, issues on the context's stream and returns once its
 * device work is done (a trace retries its hit stream inside).  Destroy a target before its context or group.
 * GPU test: tests/test_gpu_texture_target.py. */
enum { AICB_TEXTURE_INCREMENTAL = 1, AICB_TEXTURE_CONSISTENT = 2 };
typedef struct aicb_texture_target aicb_texture_target;
typedef struct aicb_texture_target_info {
    uint32_t width, height;
    uint32_t strategy;             /* AICB_TEXTURE_INCREMENTAL or AICB_TEXTURE_CONSISTENT */
    uint32_t _pad;
    uint64_t dirty_pixels;
    uint64_t next_pick;            /* the pick position: PixelPicker's count of picks, or Consistent's `next` */
    uint64_t cycle_length;
} aicb_texture_target_info;
aicb_status aicb_texture_target_create(aicb_ctx *, uint32_t width, uint32_t height, int strategy,
                                       aicb_texture_target **out);
void aicb_texture_target_destroy(aicb_texture_target *);
aicb_status aicb_texture_target_resize(aicb_texture_target *, uint32_t width, uint32_t height);
aicb_status aicb_texture_target_mark_dirty(aicb_texture_target *);
aicb_status aicb_texture_target_trace(aicb_texture_target *, const aicb_layer *world_or_null,
                                      const aicb_layer *ui_or_null, const float backdrop_rgba[4],
                                      const float no_world_rgba[4], const double depth_transform[16], size_t n,
                                      size_t *n_traced_or_null, aicb_render_info *info_or_null);
aicb_status aicb_texture_target_state(const aicb_texture_target *, aicb_texture_target_info *out);
aicb_status aicb_texture_target_picks(aicb_texture_target *, uint64_t start, size_t n, uint32_t *out);
aicb_status aicb_texture_target_buffers(aicb_texture_target *, void **d_rgba16f, void **d_depth);
aicb_status aicb_texture_target_read(aicb_texture_target *, uint16_t (*rgba16f_or_null)[4], float *depth_or_null,
                                     size_t n);

/* The texture target on a device group, with the same semantics, state and results: the order and both targets live
 * on device 0; a batch is cut into contiguous ranges of whole 32-pick warps, one per device, as
 * aicb_group_render_layers_texture cuts a pixel list, every device computes its own picks (reading device 0's order
 * over peer access) and stores its texels straight into device 0's targets.  The layers must be scenes of the target's
 * group.  Every call holds every context of the group. */
typedef struct aicb_group_texture_target aicb_group_texture_target;
aicb_status aicb_group_texture_target_create(aicb_group *, uint32_t width, uint32_t height, int strategy,
                                             aicb_group_texture_target **out);
void aicb_group_texture_target_destroy(aicb_group_texture_target *);
aicb_status aicb_group_texture_target_resize(aicb_group_texture_target *, uint32_t width, uint32_t height);
aicb_status aicb_group_texture_target_mark_dirty(aicb_group_texture_target *);
aicb_status aicb_group_texture_target_trace(aicb_group_texture_target *, const aicb_group_layer *world_or_null,
                                            const aicb_group_layer *ui_or_null, const float backdrop_rgba[4],
                                            const float no_world_rgba[4], const double depth_transform[16], size_t n,
                                            size_t *n_traced_or_null, aicb_render_info *info_or_null);
aicb_status aicb_group_texture_target_state(const aicb_group_texture_target *, aicb_texture_target_info *out);
aicb_status aicb_group_texture_target_picks(aicb_group_texture_target *, uint64_t start, size_t n, uint32_t *out);
aicb_status aicb_group_texture_target_buffers(aicb_group_texture_target *, void **d_rgba16f, void **d_depth);
aicb_status aicb_group_texture_target_read(aicb_group_texture_target *, uint16_t (*rgba16f_or_null)[4],
                                           float *depth_or_null, size_t n);

/* == SpaceRaytracer::trace_ray (sr.rs:113-120) for a batch of explicit rays:
 * origin_dir[i] = {ox,oy,oz,dx,dy,dz}. Output as aicb_render_colorbuf. */
aicb_status aicb_trace_rays(aicb_scene *, const double (*origin_dir)[6], size_t n, const aicb_options *,
                            float (*out_colorbuf)[4], double *depth_or_null, aicb_hit *hit_or_null,
                            uint32_t *steps_or_null, aicb_render_info *info_or_null);

/* ---------------------------------------------------------------------------------------------
 * Camera construction (host only, no GPU): Camera::new + look_at_y_up + compute_matrices
 * (camera_struct.rs:86-110, 387-416, 459-471); eye_for_look_at (all-is-cubes/src/camera.rs:34-40).
 * ------------------------------------------------------------------------------------------- */
/* fov_y_degrees and view_distance are repaired like GraphicsOptions::repair. nominal_* is the
 * Viewport nominal size (aspect ratio); fb_* the framebuffer size. */
aicb_status aicb_camera_look_at(const double eye[3], const double target[3], double fov_y_degrees,
                                double view_distance, double nominal_width, double nominal_height,
                                uint32_t fb_width, uint32_t fb_height, float exposure, aicb_camera *out);
/* General form: rotation quaternion (i,j,k,r) + translation of the eye-to-world ViewTransform. */
aicb_status aicb_camera_from_view(const double rotation_ijkr[4], const double translation[3],
                                  double fov_y_degrees, double view_distance, double nominal_width,
                                  double nominal_height, uint32_t fb_width, uint32_t fb_height,
                                  float exposure, aicb_camera *out);
void aicb_eye_for_look_at(const aicb_aab *bounds, const double direction[3], double out_eye[3]);
/* Camera::project_ndc_into_world for one NDC point (host, for tests): out = origin xyz, dir xyz. */
void aicb_camera_project_ndc(const aicb_camera *, double ndc_x, double ndc_y, double out_origin_dir[6]);
/* ViewTransform::to_transform (RigidTransform3D::to_transform: rotation.to_transform().then(translation.to_transform()))
 * of an eye's view transform {rotation (i, j, k, r), translation}: m11..m44 in the row-vector convention of
 * aicb_camera, the eye-to-world matrix aicb_step_exposure takes.  Host only. */
void aicb_view_transform_matrix(const double rotation_ijkr[4], const double translation[3], double out[16]);

/* ---------------------------------------------------------------------------------------------
 * The cursor: cursor_raycast (all-is-cubes/src/character/cursor.rs:26-107) and StandardCameras::project_cursor
 * (all-is-cubes-render/src/camera/stdcam.rs:357-389) over a scene's cells on the device, for a batch of queries.
 * One query finds the first cube of Raycaster::new(origin, normalize(direction)).within(bounds, false) whose block is
 * selectable (AICB_BLOCK_NOT_SELECTABLE clear, not is_air) and whose voxels let the ray select it: a single voxel
 * (Evoxels::One, or a resolution-1 block, whose voxel outside its bounds is Evoxel::AIR) by its AICB_VOXEL_* flag;
 * otherwise the first voxel of recursive_raycast(...).within(voxel_bounds, true) that is selectable, face_selected
 * being the face of that cast's first step.  The walk stops at the first step with t_distance > maximum_distance.
 * Nothing of the scene changes: not the host mirror of the block ids (no call here rebuilds it), the light, the
 * queue, the set of changed cubes, nor an asynchronous frame in flight (aicb_render_finish reports it unchanged).
 * ------------------------------------------------------------------------------------------- */
#define AICB_CURSOR_NONE 0xFFFFFFFFu      /* block_id of a query that selected nothing; preceding_block_id of WITHIN */
#define AICB_CURSOR_OUTSIDE 0xFFFFFFFEu   /* preceding_block_id of a preceding cube outside the bounds (AIR there) */
/* Cursor + its CubeSnapshots (cursor.rs:111-149), 80 bytes.  A query that selects nothing has block_id and
 * preceding_block_id AICB_CURSOR_NONE and every other byte 0. */
typedef struct aicb_cursor {
    double point_entered[3];       /* step.intersection_point(ray), the ray's direction normalised */
    double distance;               /* PositiveSign::new_clamped(step.t_distance()) */
    int32_t cube[3];               /* the selected cube */
    int32_t preceding_cube[3];     /* step.cube_behind(); = cube when face_entered is AICB_FACE_WITHIN */
    uint32_t block_id;             /* the Space's block id at `cube` */
    uint32_t preceding_block_id;   /* its id; AICB_CURSOR_OUTSIDE outside the bounds; AICB_CURSOR_NONE when WITHIN */
    uint8_t light[4];              /* Space::get_light(cube), aicb_light_download's format (PackedLight::ONE under
                                      LightPhysics::None) */
    uint8_t preceding_light[4];    /* get_light(preceding_cube): BlockSky::light_outside beyond the bounds; 0 when
                                      WITHIN */
    uint8_t face_entered, face_selected;   /* Face7 (AICB_FACE_*) */
    uint8_t layer;                 /* aicb_project_cursor: 0 nothing, 1 the UI layer, 2 the world layer; else 0 */
    uint8_t _pad[5];
} aicb_cursor;
/* cursor_raycast for n rays {ox,oy,oz,dx,dy,dz}, with maximum_distance max_distance_or_null[i] (NULL: every ray
 * f64::INFINITY; NaN sets no limit, as `t_distance > NaN` never holds).  Returns once `out` is written.
 * AICB_ERR_INVALID with nothing written: NULL rays or out with n > 0.  n == 0 does nothing. */
aicb_status aicb_cursor_raycast(aicb_scene *, const double (*origin_dir)[6], const double *max_distance_or_null,
                                size_t n, aicb_cursor *out);
/* The same with the rays (8-byte aligned), the distances and `out` (8-byte aligned) in device memory of the scene's
 * device, issued on `stream` (NULL: the context's) with the device calls' ordering (aicb_scene_update_cubes_device):
 * it reads the rays after the work queued there before it, and work queued there afterwards sees `out`.  It does not
 * synchronise on one context.  Pointers are checked as those calls check them (AICB_ERR_INVALID). */
aicb_status aicb_cursor_raycast_device(aicb_scene *, const double (*d_origin_dir)[6], const double *d_max_distance_or_null,
                                       size_t n, aicb_cursor *d_out, void *stream);
/* project_cursor for n NDC points: per point, the UI layer's cursor_raycast with f64::INFINITY, then if it selected
 * nothing the world layer's with world_max_distance (the reference hard-codes 6.0); each layer's ray is
 * Camera::project_ndc_into_world(ndc) of its camera (aicb_camera_project_ndc, as frames compute it), and `layer` says
 * which answered.  Only the layers' scenes and cameras are read.  Either layer may be NULL.  AICB_ERR_INVALID with
 * nothing written: NULL ndc or out with n > 0, a layer without a scene or camera, or layers on two contexts. */
aicb_status aicb_project_cursor(const aicb_layer *world_or_null, const aicb_layer *ui_or_null, const double (*ndc)[2],
                                size_t n, double world_max_distance, aicb_cursor *out);
/* The group forms: outputs bit-identical to one context's.  The batch is cut into ranges of whole warps, one per
 * replica, as aicb_group_trace_rays cuts its rays; each replica walks its own cells and stores into device 0.  The
 * device form's buffers are device 0's memory; a group call returns once every replica's part is done.
 * GPU test: tests/test_gpu_cursor.py. */
aicb_status aicb_group_cursor_raycast(aicb_group_scene *, const double (*origin_dir)[6],
                                      const double *max_distance_or_null, size_t n, aicb_cursor *out);
aicb_status aicb_group_cursor_raycast_device(aicb_group_scene *, const double (*d_origin_dir)[6],
                                             const double *d_max_distance_or_null, size_t n, aicb_cursor *d_out,
                                             void *stream);
aicb_status aicb_group_project_cursor(const aicb_group_layer *world_or_null, const aicb_group_layer *ui_or_null,
                                      const double (*ndc)[2], size_t n, double world_max_distance, aicb_cursor *out);

/* ---------------------------------------------------------------------------------------------
 * Bodies: step_one_body (all-is-cubes/src/physics/step.rs:316-590) against a scene's cells on the device, for a batch
 * of bodies, with the collision functions of physics/collision.rs:100-249.  A block's collision is derived when it is
 * placed, as compute_derived derives uniform_collision (block/eval/derived.rs:85-104, 159-190): Hard, None, or mixed,
 * in which case its voxels' AICB_VOXEL_NO_COLLISION flags decide; an is_air block is None.  Arithmetic is f64 without
 * contraction, as the reference's.  Nothing of the scene changes (as the cursor calls: no host mirror rebuild, no light
 * state, no frame in flight).
 * ------------------------------------------------------------------------------------------- */
/* Body (physics/body.rs:38-90) without its look direction, 152 bytes.  Boxes are {lower xyz, upper xyz}.  `occupying`
 * should contain `position` (Body's invariant), but a crush can leave it not containing it, as the reference's
 * crush_if_colliding can ("TODO: stop if we would lose the occupying-contains-position property"), so a body a step
 * returns is always a body a step takes. */
typedef struct aicb_body {
    double position[3];
    double velocity[3];
    double collision_box[6];       /* relative to position */
    double occupying[6];           /* absolute; should contain position (see above), need not */
    uint8_t flying, noclip;
    uint8_t _pad[6];
} aicb_body;
enum { AICB_CONTACT_NONE = 0, AICB_CONTACT_BLOCK = 1, AICB_CONTACT_VOXEL = 2 };
/* Contact (physics/contact.rs:31-48), 28 bytes: Block(CubeFace { cube, face }) or Voxel { cube, resolution,
 * voxel: CubeFace }; AICB_CONTACT_NONE stands for Option::None where a contact is optional.  `voxel` and
 * `resolution` are 0 unless kind is AICB_CONTACT_VOXEL. */
typedef struct aicb_contact {
    int32_t cube[3];
    int32_t voxel[3];
    uint8_t kind;                  /* AICB_CONTACT_* */
    uint8_t face;                  /* Face7 (AICB_FACE_*) */
    uint8_t resolution;
    uint8_t _pad;
} aicb_contact;
/* MoveSegment (step.rs:231-241), 56 bytes. */
typedef struct aicb_move_segment {
    double delta_position[3];
    aicb_contact stopped_by;       /* kind AICB_CONTACT_NONE: not stopped */
    uint32_t _pad;
} aicb_move_segment;
/* UncrushInfo (step.rs:281-295) */
enum { AICB_UNCRUSH_NOT_NEEDED = 0, AICB_UNCRUSH_NOT_POSSIBLE = 1, AICB_UNCRUSH_COMPLETE = 2,
       AICB_UNCRUSH_PARTIAL = 3 };
#define AICB_AXIS_NONE 0xFFu
/* aicb_body_step_info::status bits.  INVALID: the body could not be a Body (a non-finite position, velocity or
 * external delta-v, a non-finite, empty or inverted collision_box, or a non-finite or inverted occupying); the body is unchanged and the rest of its info is zero.  NO_PENETRATION and SLIDING_UNFINISHED
 * are the reference's panics "collision but found no penetration" and "sliding collision loop did not finish";
 * CRUSH_UNFINISHED is a crush where the reference would not return: a shrink that leaves the box as it was (the
 * same box meets the same contact forever), or more shrinks than a finishing crush can take (four per plane of
 * resolution 128 that each face of the box could cross, plus 64).  With
 * any of the three the body is unchanged and its info holds only the status.  CONTACTS_TRUNCATED: the contact set
 * held more than max_contacts contacts; the step is unaffected. */
#define AICB_BODY_INVALID 1u
#define AICB_BODY_CONTACTS_TRUNCATED 2u
#define AICB_BODY_NO_PENETRATION 4u
#define AICB_BODY_SLIDING_UNFINISHED 8u
#define AICB_BODY_CRUSH_UNFINISHED 16u
/* BodyStepDetails (step.rs:160-215) and the size of the body's ContactSet, 312 bytes. */
typedef struct aicb_body_step_info {
    aicb_move_segment move_segments[3];
    double push_out[3];            /* valid if has_push_out */
    double initial_crush[6];       /* CrushInfo, a FaceMap: NX, NY, NZ, PX, PY, PZ */
    double delta_v[3];
    aicb_contact already_colliding;   /* the last Within contact of the move, or kind AICB_CONTACT_NONE */
    uint32_t n_contacts;           /* the ContactSet's true size */
    uint32_t status;               /* AICB_BODY_* bits */
    uint8_t quiescent;
    uint8_t has_push_out;
    uint8_t uncrush;               /* AICB_UNCRUSH_* */
    uint8_t uncrush_axes[3];       /* PARTIAL: first, second, third (0 X, 1 Y, 2 Z, AICB_AXIS_NONE: absent) */
    uint8_t _pad[6];
} aicb_body_step_info;
/* step_one_body(body, tick, external_delta_v, Some(space)) for n bodies, in place: what the reference leaves in each
 * body, its BodyStepDetails in info_or_null[i], and its ContactSet, each contact once in first-insertion order, in
 * contacts_or_null[i * max_contacts ...] (n_contacts of them, at most max_contacts).  external_delta_v_or_null: NULL is
 * zero.  gravity: SpacePhysics::gravity.  dt: Tick::delta_t in seconds, finite and in (0, 1] (a paused tick is not
 * a step).  A body with noclip moves without collision and without gravity, as the reference's.
 * AICB_ERR_INVALID with nothing written: a NULL bodies with n > 0, a non-finite gravity, a dt out of range, or any
 * body the reference could not hold (see AICB_BODY_INVALID).  Returns once the bodies and outputs are written. */
aicb_status aicb_step_bodies(aicb_scene *, aicb_body *bodies, const double (*external_delta_v_or_null)[3], size_t n,
                             double dt, const double gravity[3], aicb_body_step_info *info_or_null,
                             aicb_contact *contacts_or_null, uint32_t max_contacts);
/* The same with bodies, external_delta_v, info and contacts (8-byte aligned) in device memory of the scene's device,
 * and gravity on the host, issued on `stream` (NULL: the context's) with the device calls' ordering
 * (aicb_cursor_raycast_device).  It does not synchronise on one context.  The scalar arguments are checked as the host
 * form checks them; a body the reference could not hold gets AICB_BODY_INVALID in its info and is left unchanged. */
aicb_status aicb_step_bodies_device(aicb_scene *, aicb_body *d_bodies, const double (*d_external_delta_v_or_null)[3],
                                    size_t n, double dt, const double gravity[3], aicb_body_step_info *d_info_or_null,
                                    aicb_contact *d_contacts_or_null, uint32_t max_contacts, void *stream);
/* The group forms: outputs bit-identical to one context's; the batch is cut into whole warps, one range per replica,
 * each replica walking its own cells and storing into device 0's buffers.  GPU test: tests/test_gpu_body_step.py. */
aicb_status aicb_group_step_bodies(aicb_group_scene *, aicb_body *bodies, const double (*external_delta_v_or_null)[3],
                                   size_t n, double dt, const double gravity[3], aicb_body_step_info *info_or_null,
                                   aicb_contact *contacts_or_null, uint32_t max_contacts);
aicb_status aicb_group_step_bodies_device(aicb_group_scene *, aicb_body *d_bodies,
                                          const double (*d_external_delta_v_or_null)[3], size_t n, double dt,
                                          const double gravity[3], aicb_body_step_info *d_info_or_null,
                                          aicb_contact *d_contacts_or_null, uint32_t max_contacts, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Automatic exposure: character::exposure::State::step (all-is-cubes/src/character/exposure.rs:67-136) over a scene's
 * cells and light on the device, for a batch of eyes.  Per tick each eye casts 10 rays from its eye-to-world transform's
 * origin through the Space (Raycaster::new(origin, direction).within(bounds, false), at most 2 * maximum_distance
 * steps, none under LightPhysics::None); a ray's sample is the luminance of get_light(cube_behind) at the first visible
 * block (Derived::visible, derived when the block is placed) whose light there is Visible, else of the sky in the ray's
 * direction.  The moving average of 100 samples sets the target exposure, and exposure_log moves towards its ln.  The
 * f32 ln and exp are correctly rounded (glibc's logf and expf where those are).  Nothing of the scene changes (as the
 * cursor calls: no host mirror rebuild, no light state, no frame in flight).
 * ------------------------------------------------------------------------------------------- */
/* exposure::State (exposure.rs:37-58), 408 bytes.  The default state is every sample 1.0f, index 0 and log 0. */
typedef struct aicb_exposure_state {
    float luminance_samples[100];
    uint32_t luminance_sample_index;   /* the last sample written; advanced as a 64-bit usize, (index + 1) % 100 */
    float exposure_log;                /* ln of the exposure */
} aicb_exposure_state;
/* State::step(space, view_transform, dt) for n eyes, in place; exposure_out_or_null[i] = State::exposure() afterwards
 * (exp(exposure_log), correctly rounded).  eye_to_world[i]: aicb_view_transform_matrix of the eye's view transform,
 * or any matrix: an origin whose w is not > 0 leaves the state unchanged, as transform_point3d's None does.
 * dt: Tick::delta_t in seconds, finite and >= 0; dt == 0 leaves every state unchanged (the reference returns early).
 * AICB_ERR_INVALID with nothing written: NULL states or eye_to_world with n > 0, or a dt out of range.  Returns once the
 * states and exposures are written. */
aicb_status aicb_step_exposure(aicb_scene *, aicb_exposure_state *states, const double (*eye_to_world)[16], size_t n,
                               double dt, float *exposure_out_or_null);
/* The same with states (4-byte aligned), matrices (8-byte aligned) and exposures (4-byte aligned) in device memory of
 * the scene's device, issued on `stream` (NULL: the context's) with the device calls' ordering
 * (aicb_cursor_raycast_device).  It does not synchronise on one context.  Pointers and dt are checked as the host
 * form checks them (AICB_ERR_INVALID). */
aicb_status aicb_step_exposure_device(aicb_scene *, aicb_exposure_state *d_states, const double (*d_eye_to_world)[16],
                                      size_t n, double dt, float *d_exposure_out_or_null, void *stream);
/* The group forms: outputs bit-identical to one context's.  The eyes are cut into ranges, one per replica; each replica
 * walks its own cells and stores into device 0's buffers.  GPU test: tests/test_gpu_exposure.py. */
aicb_status aicb_group_step_exposure(aicb_group_scene *, aicb_exposure_state *states, const double (*eye_to_world)[16],
                                     size_t n, double dt, float *exposure_out_or_null);
aicb_status aicb_group_step_exposure_device(aicb_group_scene *, aicb_exposure_state *d_states,
                                            const double (*d_eye_to_world)[16], size_t n, double dt,
                                            float *d_exposure_out_or_null, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Characters' eyes on the device: step_eye_position (all-is-cubes/src/character/eye.rs:90-121), compute_view_transform
 * (eye.rs:187-203) and the world camera StandardCameras::update builds from it (stdcam.rs:237-256: set_view_transform,
 * compute_matrices, set_measured_exposure), for a batch of eyes.  With aicb_step_bodies_device and
 * aicb_step_exposure_device, a tick of many characters is one stream of device calls with no host wait:
 *   bodies, then exposure, then eyes, then eye views, then cursor and frames (INTEGRATION §2p).
 * The body's look rotation comes in as a quaternion (aicb_look_rotation on the host): yaw and pitch come from input,
 * and their sine and cosine are glibc's, which the device could not reproduce bit for bit.  Nothing of the scene is
 * read or changed (no host mirror rebuild, no light state, no frame in flight); the scene fixes the device and the
 * context's stream.
 * ------------------------------------------------------------------------------------------- */
/* CharacterEye and PreviousBodyVelocity (eye.rs:38-57), 72 bytes.  All zeros is CharacterEye::default().
 * previous_body_velocity is the body's velocity before this tick's body step: aicb_step_eyes_device stores the body's
 * velocity there after each step, which is what the next tick's record_previous_velocity (eye.rs:83-87) reads as long
 * as nothing else changes the body between ticks.  A host that changes a velocity outside the body step (a teleport,
 * a jump added on a paused tick) writes previous_body_velocity too. */
typedef struct aicb_eye {
    double displacement_pos[3];
    double displacement_vel[3];
    double previous_body_velocity[3];
} aicb_eye;
/* What the world camera takes from GraphicsOptions and the Viewport, shared by a batch, 48 bytes.  fov_y_degrees and
 * view_distance are repaired as aicb_camera_from_view repairs them.  The exposure rule (set_measured_exposure,
 * camera_struct.rs:169-181): automatic_exposure == 0 is ExposureOption::Fixed(fixed_exposure); lighting_display is an
 * AICB_LIGHT_* value. */
typedef struct aicb_eye_view_params {
    double fov_y_degrees;
    double view_distance;
    double nominal_width;
    double nominal_height;
    uint32_t fb_width, fb_height;
    float fixed_exposure;
    uint8_t automatic_exposure;
    uint8_t lighting_display;
    uint8_t _pad[2];
} aicb_eye_view_params;
/* aicb_eye_views_device status: the projection-view matrix has no inverse (the reference panics,
 * camera_struct.rs:416); nothing else of that eye is written. */
#define AICB_EYE_NOT_INVERTIBLE 1u
/* Body::look_rotation (physics/body.rs:285-292): around_x(-pitch in radians).then(around_y(-yaw in radians)), with
 * glibc's sin and cos, as (i, j, k, r).  Host only. */
void aicb_look_rotation(double yaw_degrees, double pitch_degrees, double out_ijkr[4]);
/* step_eye_position for one stepped tick, eye i against body i, in place: the displacement spring moves by the
 * change of the body's velocity since previous_body_velocity, in uncontracted f64, with 1e21^dt and 1e-9^dt computed
 * once by the host's pow; then previous_body_velocity = the body's velocity.  A paused tick is no step: do not call
 * it then.  dt: finite and in (0, 1], as aicb_step_bodies takes it.  Eyes and bodies (8-byte aligned) are device
 * memory of the scene's device; the call is issued on `stream` (NULL: the context's) with the device calls' ordering
 * (aicb_cursor_raycast_device) and does not synchronise.  AICB_ERR_INVALID with nothing issued: NULL eyes or bodies
 * with n > 0, a pointer that is not the scene's device memory or is misaligned, or a dt out of range. */
aicb_status aicb_step_eyes_device(aicb_scene *, aicb_eye *d_eyes, const aicb_body *d_bodies, size_t n, double dt,
                                  void *stream);
/* compute_view_transform and the world camera's update for eye i, every tick (paused or not), after the exposure
 * step.  Rotation i is d_rotations[i] (i, j, k, r); the translation is body i's position + eye i's displacement.
 * Writes, for each output that is not NULL:
 *   eye_to_world[i]: aicb_view_transform_matrix of {rotation, translation}, the matrix the next tick's
 *     aicb_step_exposure_device takes (a fresh eye's all-zero matrix leaves its first exposure step a no-op, as
 *     view_transform: None does);
 *   cameras[i]: the whole record, inverse_projection_view as aicb_camera_from_view gives it for the same rotation,
 *     translation and params, fb_width and fb_height from params, _pad 0, and the exposure of set_measured_exposure:
 *     under Fixed the fixed value; under automatic exposure d_exposures[i] (the aicb_step_exposure_device output)
 *     when it is not NaN and not negative (-0 as +0), or 1 for it under AICB_LIGHT_NONE; an invalid measurement or
 *     NULL d_exposures keeps the entry's exposure;
 *   look_rays[i]: {origin xyz, direction xyz} of the new camera at the screen centre, aicb_camera_project_ndc at
 *     (0, 0): with aicb_cursor_raycast_device and a distance of 6, what the character is looking at;
 *   status[i]: 0, or AICB_EYE_NOT_INVERTIBLE with nothing else of the eye written.
 * Rotations, eyes, bodies, matrices, cameras and rays are 8-byte aligned, exposures and statuses 4-byte aligned,
 * device memory of the scene's device; the call is issued as aicb_step_eyes_device is.  AICB_ERR_INVALID with nothing
 * issued: a NULL params, NULL eyes, bodies or rotations with n > 0, or a pointer the device calls reject. */
aicb_status aicb_eye_views_device(aicb_scene *, const aicb_eye *d_eyes, const aicb_body *d_bodies,
                                  const double (*d_rotations)[4], const float *d_exposures_or_null, size_t n,
                                  const aicb_eye_view_params *params, double (*d_eye_to_world_or_null)[16],
                                  aicb_camera *d_cameras_or_null, double (*d_look_rays_or_null)[6],
                                  uint32_t *d_status_or_null, void *stream);
/* The group forms run on device 0 with device 0's buffers, and their outputs are one context's bytes.  They do not
 * synchronise either.  GPU test: tests/test_gpu_eyes.py. */
aicb_status aicb_group_step_eyes_device(aicb_group_scene *, aicb_eye *d_eyes, const aicb_body *d_bodies, size_t n,
                                        double dt, void *stream);
aicb_status aicb_group_eye_views_device(aicb_group_scene *, const aicb_eye *d_eyes, const aicb_body *d_bodies,
                                        const double (*d_rotations)[4], const float *d_exposures_or_null, size_t n,
                                        const aicb_eye_view_params *params, double (*d_eye_to_world_or_null)[16],
                                        aicb_camera *d_cameras_or_null, double (*d_look_rays_or_null)[6],
                                        uint32_t *d_status_or_null, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Light propagation (secondary path): replaces Mutation::set x n + evaluate_light(epsilon)
 * (space.rs:1346-1352, 1496-1527; space/light/updater.rs:181-363).
 * ------------------------------------------------------------------------------------------- */
/* The static light-ray chart (space/light/chart/generator.rs:49-215) as the flat prefix tree the kernels
 * walk: 6 f32 weights + 6 child indices (0 = none) per node, root = 0.  Returns the node count
 * (114 779); either pointer may be NULL.  Host only. */
uint32_t aicb_light_chart(float *weights_or_null, uint32_t *children_or_null);
/* The same chart the way the kernels walk it: in depth-first preorder (children in Face6 order, the order walk_ray_tree
 * recurses in, updater.rs:500) and cut into chains — maximal paths of single-child nodes, which carry bit-identical
 * weights; a chain's nodes are consecutive in preorder and chains are numbered breadth first.  Host only; any pointer
 * may be NULL.  preorder[i] = index in aicb_light_chart's numbering of the i-th node in preorder (node count entries);
 * chains[c] = {first node (preorder), nodes, child chains, first child chain, parent's branch slot or 0xffff, own
 * branch slot or 0xffff}; euler = the Euler tour of the chain tree, chain | 0x8000 for the chain's exit (n_euler
 * entries = 2 * n_chains): the order in which the terms of a walk are added.  Returns the number of chains (1043). */
uint32_t aicb_light_chart_chains(uint32_t *preorder_or_null, uint32_t (*chains_or_null)[6], uint16_t *euler_or_null);
/* LightStorage::fast_evaluate_light (updater.rs:537-582): column-sweep initial guess + queue seeding. */
aicb_status aicb_light_fast_evaluate(aicb_scene *);
/* LightStorage::compute_light (updater.rs:368-418) for explicit cubes against the current field; does not
 * store anything (parity tests). out[i] = PackedLight::as_texel. */
aicb_status aicb_light_compute(aicb_scene *, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]);
/* Mutation::evaluate_light(epsilon) (space.rs:1496-1527): relax until the highest queued priority is
 * <= Priority::from_difference(epsilon). */
aicb_status aicb_light_evaluate(aicb_scene *, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                                uint64_t *chart_node_visits_or_null);
/* LightUpdatesInfo (space/light/updater.rs:970-984) of one step. */
typedef struct aicb_light_updates_info {
    uint64_t update_count;          /* compute_light + apply_light_update calls this step */
    uint64_t queue_count;           /* cubes queued after the step */
    uint8_t max_update_difference;  /* largest difference_priority applied this step */
    uint8_t max_queue_priority;     /* highest queued Priority after the step; 0 (Priority::MIN) when empty */
    uint8_t _pad[6];
} aicb_light_updates_info;
/* LightStorage::update_light_from_queue (space/light/updater.rs:180-290) with a budget of cube updates: the light step
 * of a tick (update_light_system, space/step.rs:341-369).  A host edits with aicb_light_edit_cubes and
 * aicb_light_edit_region (or the queue calls below), calls this with the tick's budget, then takes the changed cubes;
 * light converges over several ticks and no tick stalls.  The call is synchronous and deterministic, and the library keeps no clock: a host with a time budget
 * turns it into a count, e.g. from aicb_light_stats' out[3] / out[0] of earlier steps.
 *   - Work: relaxation rounds on the queue, as aicb_light_evaluate runs them, until max_updates cube updates are made
 *     or the queue is empty.  info->update_count = min(max_updates, the updates the queue offered); a cube re-queued
 *     and updated again counts twice.  Every queued priority >= 1 is eligible (aicb_light_evaluate(0) leaves
 *     priority-1 entries, which only a host's aicb_light_queue_region(..., 1) creates).  max_updates == 0 runs no round
 *     and fills info; UINT64_MAX is the reference's `budget: None`.
 *   - Which cubes: a round whose band (the cubes within 16 priority levels of the round's highest) fits in the budget
 *     left is aicb_light_evaluate's round.  A round that does not fit takes the budget's worth of the band: by
 *     priority, highest first, and within the priority where the budget ends, lowest Z-major index first.  So the set
 *     of cubes a step updates depends only on the queue.
 *   - A round stays whole: its cubes' results are stored, the set of changed cubes updated and their dependencies
 *     re-queued (on a group, the replicas updated) before the call returns.
 *   - info_or_null: queue_count and max_queue_priority are exact, as aicb_light_download_queue would report them.
 *     aicb_light_stats reads as after aicb_light_evaluate, with out[0] == update_count.
 * AICB_ERR_INVALID, with nothing changed: a NULL scene or LightPhysics::None.  GPU test: tests/test_gpu_light_step.py. */
aicb_status aicb_light_update_from_queue(aicb_scene *, uint64_t max_updates, aicb_light_updates_info *info_or_null);
/* Mutation::set(cubes[i], new_ids[i]) for i = 0 .. n-1, in list order (space.rs:1346-1352 -> side_effects_of_set ->
 * modified_cube_needs_update, space/light/updater.rs:135-173), on a scene whose light the library computes: the
 * SpaceChange::CubeBlock batch of a tick.
 *   - An entry is changing if its id differs from the block its cube holds at that point of the list (Mutation::set of
 *     the same block changes nothing); a cube may be named any number of times.  The cells, the host mirror, the
 *     texels, the queue and the set of changed cubes end byte for byte as the entries applied one by one leave them.
 *   - Each changing entry applies the light rule: a block opaque for light stores OPAQUE, cancels the cube's queued
 *     update and puts the cube into the set of changed cubes; any other block queues the cube at
 *     Priority::NEWLY_VISIBLE; every in-bounds face neighbour whose own face toward the cube is not opaque is queued at
 *     NEWLY_VISIBLE.  A cube set to an opaque block and back keeps its OPAQUE texel and is queued, as in the reference.
 *   - *n_changed_or_null: the number of changing entries, the SpaceChange::CubeBlock the reference sends for the list.
 *   - Nothing propagates: aicb_light_evaluate or aicb_light_update_from_queue follows when the host wants the light to
 *     move.  aicb_light_stats is left as it was.
 *   - The call is ordered like aicb_light_edit_region: behind the cube updates queued on the context, before any later
 *     render, and it returns once its writes are done.  The rule runs on the device against the final cells.
 * n == 0 changes nothing and reports 0.  AICB_ERR_INVALID, with nothing changed: NULL cubes or new_ids with n > 0, any
 * cube out of bounds, an id >= the table's size, n >= 2^32, or LightPhysics::None.
 * GPU test: tests/test_gpu_light_edit_cubes.py. */
aicb_status aicb_light_edit_cubes(aicb_scene *, const int32_t (*cubes)[3], const uint16_t *new_ids, size_t n,
                                  size_t *n_changed_or_null);
/* aicb_light_edit_cubes, then Mutation::evaluate_light(epsilon) as aicb_light_evaluate runs it. */
aicb_status aicb_light_edit_and_propagate(aicb_scene *, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                          size_t n_edits, uint8_t epsilon, uint64_t *updates_done,
                                          uint8_t *max_diff);
/* The light side of SpaceChange::BlockEvaluation: after aicb_scene_update_blocks gave `indices` new definitions, apply
 * Mutation::set's light rule (side_effects_of_set -> modified_cube_needs_update, space.rs:499-531,
 * space/light/updater.rs:135-173) to every cube that holds one of them, with the block's current definition, then
 * evaluate_light(epsilon) as aicb_light_edit_and_propagate does.  The same-block skip of Mutation::set does not apply:
 *   - a block opaque for light (every face opaque, no emission): its cubes' texels become OPAQUE, even over OPAQUE,
 *     their queued updates are cancelled and they enter the set of changed cubes;
 *   - any other block: its cubes are queued at Priority::NEWLY_VISIBLE;
 *   - either way, every in-bounds face neighbour of the cube whose own face toward it is not opaque is queued at
 *     NEWLY_VISIBLE.
 * The cubes are found on the device by a scan of the cells (2 or 4 bytes per cube), ordered behind the cube updates
 * queued on the context.  Duplicates are allowed; an index no cube holds adds nothing; n == 0 only relaxes.
 * AICB_ERR_INVALID, with nothing changed: NULL with n > 0, an index >= the table's size, or LightPhysics::None.
 * The counters of aicb_light_stats are the propagation's (the scan is not in its device time).  aicb_scene_update_blocks
 * itself does not touch light.  GPU test: tests/test_gpu_light_relight.py. */
aicb_status aicb_light_relight_blocks(aicb_scene *, const uint16_t *indices, size_t n, uint8_t epsilon,
                                      uint64_t *updates_done, uint8_t *max_diff);
aicb_status aicb_light_download(aicb_scene *, uint8_t (*out)[4], size_t n_texels);
/* Mutation::fill / fill_uniform over a region smaller than the bounds (space.rs:1392-1412, 1455-1479) on a scene whose
 * light the library computes: Mutation::set for every cube of `region` in interior_iter order.  The arguments are
 * aicb_scene_update_region's; a cube the fill leaves alone is passed the id it already holds (Mutation::set of the same
 * block changes nothing).  The cells and the host mirror take the ids, and every cube whose block changes gets
 * Mutation::set's light rule (modified_cube_needs_update, space/light/updater.rs:135-173) as
 * aicb_light_edit_and_propagate applies it: a block opaque for light stores OPAQUE, cancels the cube's queued update and
 * puts the cube into the set of changed cubes; any other block queues the cube at Priority::NEWLY_VISIBLE; every
 * in-bounds face neighbour whose own face toward the cube is not opaque is queued at NEWLY_VISIBLE.  The rule runs on
 * the device against the box's final cells, which leaves the queue and the texels the cube-by-cube order leaves.
 * Nothing propagates: aicb_light_evaluate follows when the host wants the light to move, as after
 * aicb_light_queue_region.  *n_changed_or_null: the cubes whose block changed.  The call returns once its writes are
 * done.  AICB_ERR_INVALID, with nothing changed: as aicb_scene_update_region, or LightPhysics::None.
 * GPU test: tests/test_gpu_region.py. */
aicb_status aicb_light_edit_region(aicb_scene *, const aicb_aab *region, const uint16_t *block_ids_or_null,
                                   uint16_t uniform_id, size_t *n_changed_or_null);
/* The light update queue across save and load.  The queue holds one priority per cube (0: not queued); an insert raises
 * a cube's priority and never lowers it (LightUpdateQueue::insert, space/light/queue.rs).  None of these calls writes a
 * texel, adds to the set of changed cubes or propagates: aicb_light_evaluate follows, as the reference's step does.
 * LightPhysics::None is AICB_ERR_INVALID, and a rejected call changes nothing.
 *   - aicb_light_queue_uninitialized: the load rule of Space::new_from_builder (space.rs:290-313).  Every cube whose
 *     texel's status byte is 0 (LightStatus::Uninitialized) is inserted at Priority::UNINIT (210), and
 *     *n_queued_or_null is the number of such cubes.  A scene created without a light volume holds only NO_RAYS, so it
 *     queues none.  A host calls it once after aicb_scene_create from a saved Space that has light (aicb_scene_create
 *     and aicb_scene_upload_light leave the queue as it is).  The scan of the volume is ordered behind the cube updates
 *     and uploads queued on the context.
 *   - aicb_light_queue_region: LightStorage::light_needs_update_in_region (space/light/updater.rs:122-133).  Every cube
 *     of region ∩ bounds is inserted at `priority`; an empty intersection does nothing.  The reference's sweep branch
 *     (more than 400 cubes) queues the same cubes at the same priority.  After SpaceChange::EveryBlock (fill_uniform
 *     over the whole Space, space.rs:1461-1474) a host calls aicb_scene_fill_uniform, then this with the bounds and 210.
 *     AICB_ERR_INVALID: a NULL region or priority 0 (Priority::MIN never enters the queue).
 *   - aicb_light_download_queue: each cube's queued priority, Z-major (aicb_light_download's order), 0 where it is not
 *     queued; *n_queued_or_null is the number of queued cubes.  The copy is ordered behind all work on the context.
 *     AICB_ERR_INVALID: a NULL output or n_texels other than the volume.  The save form of a Space
 *     (Serialize for space::Read, save/conversion.rs:773-785) is aicb_light_download's texels with the status byte set
 *     to 0 (Uninitialized) wherever the priority is > 0, and r, g, b kept.
 * GPU test: tests/test_gpu_light_resume.py. */
aicb_status aicb_light_queue_uninitialized(aicb_scene *, size_t *n_queued_or_null);
aicb_status aicb_light_queue_region(aicb_scene *, const aicb_aab *region, uint8_t priority);
aicb_status aicb_light_download_queue(aicb_scene *, uint8_t *priorities, size_t n_texels, size_t *n_queued_or_null);
/* Counters of the last propagation (aicb_light_evaluate / aicb_light_edit_and_propagate / aicb_light_relight_blocks)
 * on this scene: out[0] cube updates (compute_light calls, updater.rs:368), out[1] chart nodes visited by them,
 * out[2] relaxation rounds queued, out[3] device time of the propagation in microseconds (CUDA events on the context's stream).
 * After aicb_light_compute: out[0] cubes computed, out[1] chart nodes visited, out[2] cubes whose walk needed more
 * term slots than the chain walk holds and took the lockstep walk instead, out[3] 0. */
aicb_status aicb_light_stats(const aicb_scene *, uint64_t out[4]);
/* SpaceChange::CubeLight (space.rs:1079-1083): the set of cubes whose light texel the light calls wrote.  A cube enters
 * it when
 *   - aicb_light_edit_cubes (or aicb_light_edit_and_propagate) sets it to a different block that is opaque for light,
 *     which stores OPAQUE even over OPAQUE (modified_cube_needs_update, space/light/updater.rs:153-161);
 *   - aicb_light_relight_blocks finds it holding a redefined block that is opaque for light (OPAQUE even over OPAQUE);
 *   - aicb_light_edit_region sets it to a different block that is opaque for light;
 *   - a relaxation round stores a value with difference_priority > 0 (apply_light_update, updater.rs:313-317);
 *   - a round writes a guess into an Uninitialized neighbour (updater.rs:335-338);
 *   - aicb_light_fast_evaluate changes its texel.  The reference announces nothing there (fast_evaluate_light has a
 *     TODO for EveryBlock); a host following the light needs the cubes all the same;
 *   - aicb_scene_set_physics reinitialises the light (every cube).
 * Nothing else adds to it: not aicb_light_compute, aicb_scene_update_cubes, aicb_scene_update_region,
 * aicb_scene_upload_light (texels the host supplied), frames, or a rejected call.  The set accumulates across calls until
 * it is taken; a scene with no light call yet has none.  LightPhysics::None is AICB_ERR_INVALID.
 * aicb_light_take_changes with both outputs and capacity >= the set's size writes each cube once, as its Z-major
 * linear index (the index into aicb_scene_desc::block_ids and light), in increasing order, with its texel as it is now
 * (aicb_light_download's format), empties the set and sets *n_taken to its size.  With both outputs NULL it empties
 * the set without copying and sets *n_taken to the number discarded: for a host that downloads the whole volume
 * instead, which is cheaper once the set exceeds half of it.  capacity < size: AICB_ERR_INVALID, *n_taken = size and
 * the set is unchanged.  Exactly one output NULL: AICB_ERR_INVALID.  Both hold the context lock; the copy is ordered
 * behind all work queued on the context. */
aicb_status aicb_light_changes_count(const aicb_scene *, size_t *n_changed);
aicb_status aicb_light_take_changes(aicb_scene *, uint32_t *indices_or_null, uint8_t (*texels_or_null)[4],
                                    size_t capacity, size_t *n_taken);
/* One ray of Space::compute_light::<LightUpdateCubeInfo> (space/light/debug.rs: LightUpdateRayInfo): a ray that ended
 * on a face opaque for light (LightBuffer::traverse, space/light/updater.rs:838-853).  trigger_cube is the cube struck,
 * value_cube the cube the ray came from, whose stored light the face reflects; value is that stored light
 * (PackedLight::as_texel, aicb_light_download's format); light_from_struck_face = the struck block's emission + its
 * face colour (clamped) * value * the colour's alpha, in f32 as the reference computes it. */
typedef struct aicb_light_ray {
    int32_t trigger_cube[3];
    int32_t value_cube[3];
    uint8_t value[4];
    float light_from_struck_face[3];
    uint32_t _pad;
} aicb_light_ray;
/* Space::compute_light::<LightUpdateCubeInfo> (space.rs:810, space/light/debug.rs) for explicit cubes against the
 * current field: aicb_light_compute with the rays that produced each result, for a host that draws them
 * (GraphicsOptions::debug_light_rays_at_cursor).  out_texels[i] is what aicb_light_compute gives for cubes[i], and
 * ray_counts[i] the number of its rays.  The rays of all cubes are packed cube after cube in list order, each cube's
 * in the reference's order (walk_ray_tree's depth-first order); an opaque cube has none.  *n_rays_total is their sum.
 * Nothing is stored: the light volume, the queue and the set of changed cubes stay as they are, and aicb_light_stats
 * reads as after aicb_light_compute on the same cubes.
 * AICB_ERR_INVALID, with nothing written but *n_rays_total: ray_capacity < the total (*n_rays_total = the total; a
 * NULL `rays` counts as capacity 0, so a first call with NULL sizes the buffer).  AICB_ERR_INVALID with nothing
 * written: NULL cubes, out_texels or ray_counts with n > 0, NULL n_rays_total, n > the volume, a cube out of bounds,
 * or LightPhysics::None.  GPU test: tests/test_gpu_light_debug.py. */
aicb_status aicb_light_compute_debug(aicb_scene *, const int32_t (*cubes)[3], size_t n, uint8_t (*out_texels)[4],
                                     aicb_light_ray *rays_or_null, size_t ray_capacity, uint32_t *ray_counts,
                                     size_t *n_rays_total);

/* The light calls above on a device group (csrc/group.cu, csrc/light.cu), with their arguments, validation, errors and
 * results: LightStorage::fast_evaluate_light / compute_light / Mutation::set x n + evaluate_light
 * (space/light/updater.rs:537-582, 368-418, 135-363; space.rs:1346-1352, 1496-1527).  Validation is against replica 0
 * before anything changes: a rejected call changes no replica.  A scene with LightPhysics::None is AICB_ERR_INVALID.
 * The first light call of a group enables device 0's peer access to every other device and checks native peer
 * atomics (AICB_ERR_UNSUPPORTED without them); a device named more than once needs neither.  Each call holds every
 * context of the group until it returns, and leaves the replicas' light volumes identical.
 * A relaxation round: device 0 gathers the round's cubes from its queue; every device computes a share of them against
 * its own replica (cubes handed out one at a time by device 0's counter); device 0 applies the results and stores the
 * 32-cube segments it wrote into every other replica (NVLink); every device re-queues the dependencies of a share of
 * the changed cubes in device 0's queue.  The group performs one context's operations, so its results meet the same
 * contract.  aicb_group_light_compute splits the cubes across the devices the same way; outputs in input order. */
aicb_status aicb_group_light_fast_evaluate(aicb_group_scene *);
aicb_status aicb_group_light_compute(aicb_group_scene *, const int32_t (*cubes)[3], size_t n, uint8_t (*out)[4]);
aicb_status aicb_group_light_evaluate(aicb_group_scene *, uint8_t epsilon, uint64_t *updates_done, uint8_t *max_diff,
                                      uint64_t *chart_node_visits_or_null);
/* aicb_light_update_from_queue on the group: validated against replica 0; the replicas are identical after it, and the
 * result is one context's. */
aicb_status aicb_group_light_update_from_queue(aicb_group_scene *, uint64_t max_updates,
                                               aicb_light_updates_info *info_or_null);
aicb_status aicb_group_light_edit_and_propagate(aicb_group_scene *, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                                size_t n_edits, uint8_t epsilon, uint64_t *updates_done,
                                                uint8_t *max_diff);
/* aicb_light_edit_cubes on the group: validated against replica 0 before any replica changes; every replica writes its
 * own cells and its own OPAQUE texels, and the scene's one host mirror is written once; device 0 alone queues and
 * records the set. */
aicb_status aicb_group_light_edit_cubes(aicb_group_scene *, const int32_t (*cubes)[3], const uint16_t *new_ids,
                                        size_t n, size_t *n_changed_or_null);
/* aicb_light_relight_blocks on the group: the indices are checked against replica 0's table; every replica scans its
 * own cells and writes its own OPAQUE texels; device 0 alone queues and records the changed cubes. */
aicb_status aicb_group_light_relight_blocks(aicb_group_scene *, const uint16_t *indices, size_t n, uint8_t epsilon,
                                            uint64_t *updates_done, uint8_t *max_diff);
/* aicb_light_edit_region on the group: validated against replica 0; every replica writes its own cells and its own
 * OPAQUE texels; device 0 alone counts the changed cubes, queues and records the set. */
aicb_status aicb_group_light_edit_region(aicb_group_scene *, const aicb_aab *region, const uint16_t *block_ids_or_null,
                                         uint16_t uniform_id, size_t *n_changed_or_null);
/* The queue calls on the group: the queue is device 0's, and aicb_group_light_queue_uninitialized scans replica 0's
 * volume (the replicas' are identical).  Validation is against replica 0 before anything changes, and each call holds
 * every context of the group. */
aicb_status aicb_group_light_queue_uninitialized(aicb_group_scene *, size_t *n_queued_or_null);
aicb_status aicb_group_light_queue_region(aicb_group_scene *, const aicb_aab *region, uint8_t priority);
aicb_status aicb_group_light_download_queue(aicb_group_scene *, uint8_t *priorities, size_t n_texels,
                                            size_t *n_queued_or_null);
/* Replica `replica` (0 .. group size - 1) of the light volume. */
aicb_status aicb_group_light_download(aicb_group_scene *, int replica, uint8_t (*out)[4], size_t n_texels);
/* aicb_light_stats of the group's last light call: counters summed over the devices; out[3] is device 0's device time
 * of the whole propagation (device 0 waits for every device in every round). */
aicb_status aicb_group_light_stats(const aicb_group_scene *, uint64_t out[4]);
/* aicb_light_changes_count / aicb_light_take_changes of the group: the set is device 0's.  Device 0 applies every round
 * and the push keeps the replicas identical, so the indices and texels are those of every replica.  Each call holds
 * every context lock of the group. */
aicb_status aicb_group_light_changes_count(const aicb_group_scene *, size_t *n_changed);
aicb_status aicb_group_light_take_changes(aicb_group_scene *, uint32_t *indices_or_null, uint8_t (*texels_or_null)[4],
                                          size_t capacity, size_t *n_taken);
/* aicb_light_compute_debug on the group: replica 0 walks every cube against its own field (the replicas' are
 * identical), with the same arguments, results and errors. */
aicb_status aicb_group_light_compute_debug(aicb_group_scene *, const int32_t (*cubes)[3], size_t n,
                                           uint8_t (*out_texels)[4], aicb_light_ray *rays_or_null, size_t ray_capacity,
                                           uint32_t *ray_counts, size_t *n_rays_total);

#ifdef __cplusplus
}
#endif
#endif /* AICB200_H */
