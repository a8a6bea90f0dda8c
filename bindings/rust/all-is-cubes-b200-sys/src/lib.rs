//! `include/aicb200.h`, item for item.  ABI version 28 (`aicb_abi_version()`).
//! Layouts are checked against the C header by `tests/test_abi.py` on the Python mirror; keep the three in step.
#![allow(non_camel_case_types)]
#![no_std]

use core::ffi::{c_char, c_int, c_void};

pub type aicb_status = c_int;
pub const AICB_OK: aicb_status = 0;
pub const AICB_ERR_INVALID: aicb_status = 1;
pub const AICB_ERR_OOM: aicb_status = 2;
pub const AICB_ERR_CUDA: aicb_status = 3;
pub const AICB_ERR_UNSUPPORTED: aicb_status = 4;
pub const AICB_ERR_BUSY: aicb_status = 5;
pub const AICB_ERR_RETRY: aicb_status = 6;

/// aicb_scene_*_blocks_device flags: light_* come from compute_derived on the device.
pub const AICB_BLOCKS_DERIVE_LIGHT: u32 = 1;

pub const AICB_TEXT_ENTERED_SPACE: i32 = -1;
pub const AICB_TEXT_EMPTY: i32 = -2;
pub const AICB_TEXT_INCOMPLETE: i32 = -3;
pub const AICB_TEXT_BLANK: i32 = -4;

pub const AICB_LAYER_NONE: i32 = 0;
pub const AICB_LAYER_WORLD: i32 = 1;
pub const AICB_LAYER_UI: i32 = 2;

/// `GridAab` (all-is-cubes-base/src/math/grid_aab.rs)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_aab {
    pub lower: [i32; 3],
    pub size: [u32; 3],
}

/// `Evoxel` without its collision (block/eval/voxel_storage.rs:41-60); `flags`: `AICB_VOXEL_*`
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_voxel {
    pub rgba: [f32; 4],
    pub emission: [f32; 3],
    pub flags: u32,
}

/// `Evoxel::selectable == false`
pub const AICB_VOXEL_NOT_SELECTABLE: u32 = 1;
/// `Evoxel::collision == BlockCollision::None` (zero: `Hard`)
pub const AICB_VOXEL_NO_COLLISION: u32 = 2;
/// `BlockAttributes::selectable == false` (an `is_air` block is never selectable)
pub const AICB_BLOCK_NOT_SELECTABLE: u32 = 1;
/// `aicb_cursor::block_id` of a query that selected nothing; `preceding_block_id` of a ray that started in the cube
pub const AICB_CURSOR_NONE: u32 = 0xFFFF_FFFF;
/// `aicb_cursor::preceding_block_id` of a preceding cube outside the bounds
pub const AICB_CURSOR_OUTSIDE: u32 = 0xFFFF_FFFE;

/// `Cursor` + its `CubeSnapshot`s (character/cursor.rs:111-149)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_cursor {
    pub point_entered: [f64; 3],
    pub distance: f64,
    pub cube: [i32; 3],
    pub preceding_cube: [i32; 3],
    pub block_id: u32,
    pub preceding_block_id: u32,
    pub light: [u8; 4],
    pub preceding_light: [u8; 4],
    pub face_entered: u8,
    pub face_selected: u8,
    pub layer: u8,
    pub _pad: [u8; 5],
}

/// `character::exposure::State` (character/exposure.rs:37-58), 408 bytes; the default state is every sample 1.0,
/// index 0 and log 0
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_exposure_state {
    pub luminance_samples: [f32; 100],
    pub luminance_sample_index: u32,
    pub exposure_log: f32,
}

impl Default for aicb_exposure_state {
    fn default() -> Self {
        Self { luminance_samples: [1.0; 100], luminance_sample_index: 0, exposure_log: 0.0 }
    }
}

/// `CharacterEye` and `PreviousBodyVelocity` (character/eye.rs:38-57), 72 bytes; all zeros is
/// `CharacterEye::default()`.  A host that changes a body's velocity outside the body step also writes
/// `previous_body_velocity`.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_eye {
    pub displacement_pos: [f64; 3],
    pub displacement_vel: [f64; 3],
    pub previous_body_velocity: [f64; 3],
}

/// What a batch of eyes' world cameras take from `GraphicsOptions` and the `Viewport`, 48 bytes;
/// `automatic_exposure == 0` is `ExposureOption::Fixed(fixed_exposure)`.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_eye_view_params {
    pub fov_y_degrees: f64,
    pub view_distance: f64,
    pub nominal_width: f64,
    pub nominal_height: f64,
    pub fb_width: u32,
    pub fb_height: u32,
    pub fixed_exposure: f32,
    pub automatic_exposure: u8,
    pub lighting_display: u8,
    pub _pad: [u8; 2],
}

/// `aicb_eye_views_device` status: the projection-view matrix has no inverse; nothing else of the eye is written.
pub const AICB_EYE_NOT_INVERTIBLE: u32 = 1;

/// `Body` (physics/body.rs:38-90) without its look direction; boxes are `[lower xyz, upper xyz]`
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_body {
    pub position: [f64; 3],
    pub velocity: [f64; 3],
    pub collision_box: [f64; 6],
    pub occupying: [f64; 6],
    pub flying: u8,
    pub noclip: u8,
    pub _pad: [u8; 6],
}

pub const AICB_CONTACT_NONE: u8 = 0;
pub const AICB_CONTACT_BLOCK: u8 = 1;
pub const AICB_CONTACT_VOXEL: u8 = 2;

/// `Contact` (physics/contact.rs:31-48), or `AICB_CONTACT_NONE` for an absent one
#[repr(C)]
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq, Hash)]
pub struct aicb_contact {
    pub cube: [i32; 3],
    pub voxel: [i32; 3],
    pub kind: u8,
    pub face: u8,
    pub resolution: u8,
    pub _pad: u8,
}

/// `MoveSegment` (physics/step.rs:231-241)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_move_segment {
    pub delta_position: [f64; 3],
    pub stopped_by: aicb_contact,
    pub _pad: u32,
}

pub const AICB_UNCRUSH_NOT_NEEDED: u8 = 0;
pub const AICB_UNCRUSH_NOT_POSSIBLE: u8 = 1;
pub const AICB_UNCRUSH_COMPLETE: u8 = 2;
pub const AICB_UNCRUSH_PARTIAL: u8 = 3;
pub const AICB_AXIS_NONE: u8 = 0xFF;
pub const AICB_BODY_INVALID: u32 = 1;
pub const AICB_BODY_CONTACTS_TRUNCATED: u32 = 2;
pub const AICB_BODY_NO_PENETRATION: u32 = 4;
pub const AICB_BODY_SLIDING_UNFINISHED: u32 = 8;
pub const AICB_BODY_CRUSH_UNFINISHED: u32 = 16;

/// `BodyStepDetails` (physics/step.rs:160-215) and the size of the body's `ContactSet`
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_body_step_info {
    pub move_segments: [aicb_move_segment; 3],
    pub push_out: [f64; 3],
    pub initial_crush: [f64; 6],
    pub delta_v: [f64; 3],
    pub already_colliding: aicb_contact,
    pub n_contacts: u32,
    pub status: u32,
    pub quiescent: u8,
    pub has_push_out: u8,
    pub uncrush: u8,
    pub uncrush_axes: [u8; 3],
    pub _pad: [u8; 6],
}

/// one entry of `Space::block_data()` as `TracingBlock::from_block` sees it (sr.rs:569-587) plus the
/// `EvaluatedBlock` members light propagation reads (block/eval/evaluated.rs:189-267)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_block_desc {
    pub resolution: u8,
    pub is_air: u8,
    pub light_opaque_faces: u8,
    pub light_visible: u8,
    pub voxel_bounds: aicb_aab,
    pub indices: *const u16,
    pub n_indices: usize,
    pub palette: *const aicb_voxel,
    pub n_palette: usize,
    pub light_face_colors: [[f32; 4]; 6],
    pub light_color: [f32; 4],
    pub light_emission: [f32; 3],
    pub flags: u32,
}

/// `compute_derived`'s light fields of one block (block/eval/derived.rs:80-216), as `aicb_block_desc`'s `light_*`
/// members take them; `opaque_faces` has bit (face - 1) per face NX..PZ.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_block_light {
    pub face_colors: [[f32; 4]; 6],
    pub color: [f32; 4],
    pub emission: [f32; 3],
    pub opaque_faces: u8,
    pub visible: u8,
    pub _pad: [u8; 2],
}

/// `Sky` (space/sky.rs:16-21): kind 0 = Uniform(colors[0]), 1 = Octants
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_sky {
    pub kind: u32,
    pub colors: [[f32; 3]; 8],
}

/// what `SpaceRaytracer::new` snapshots (sr.rs:64-88)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_scene_desc {
    pub bounds: aicb_aab,
    pub block_ids: *const u16,
    pub light: *const [u8; 4],
    pub blocks: *const aicb_block_desc,
    pub n_blocks: usize,
    pub sky: aicb_sky,
    pub light_max_distance: u8,
    pub _pad: [u8; 7],
}

/// what `Camera::project_ndc_into_world` needs (camera_struct.rs:238-257)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_camera {
    pub inverse_projection_view: [f64; 16],
    pub fb_width: u32,
    pub fb_height: u32,
    pub exposure: f32,
    pub _pad: u32,
}

/// the `GraphicsOptions` fields that affect pixels (graphics_options.rs:28-150)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_options {
    pub fog: u8,
    pub lighting_display: u8,
    pub transparency: u8,
    pub antialiasing_always: u8,
    pub tone_mapping: u8,
    pub debug_pixel_cost: u8,
    pub include_sky: u8,
    pub bounce_samples: u8,
    pub transparency_threshold: f32,
    pub maximum_intensity: f32,
    pub view_distance: f64,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_shard {
    pub strip_rows: u32,
    pub index: u32,
    pub count: u32,
}

/// `ImageInfo` / `RaytraceInfo` (renderer.rs:609-646, sr.rs:520-522) plus device timing
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_render_info {
    pub cubes_traced: u64,
    pub rays: u64,
    pub algorithmic_bytes: u64,
    pub counters: [u64; 6],
    pub kernel_ms: f32,
    pub flaws: u16,
    pub ray_order: u16,
    pub stage_ms: [f32; 4],
}

/// `Position` of the first hit (hit.rs:92-101)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_hit {
    pub cube: [i32; 3],
    pub voxel: [i32; 3],
    pub resolution: i32,
    pub face: i32,
}

/// one ray of `Space::compute_light::<LightUpdateCubeInfo>`: `LightUpdateRayInfo` (all-is-cubes/src/space/light/debug.rs)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_light_ray {
    pub trigger_cube: [i32; 3],
    pub value_cube: [i32; 3],
    pub value: [u8; 4],
    pub light_from_struck_face: [f32; 3],
    pub _pad: u32,
}

/// `LightUpdatesInfo` (all-is-cubes/src/space/light/updater.rs:970-984) of one light step
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_light_updates_info {
    pub update_count: u64,
    pub queue_count: u64,
    pub max_update_difference: u8,
    pub max_queue_priority: u8,
    pub _pad: [u8; 6],
}

/// one pixel of the terminal's frame: `ColorCharacterBuf::output` (all-is-cubes-desktop/src/terminal.rs:355-366)
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_terminal_pixel {
    pub rgba: [f32; 4],
    pub text: i32,
    pub layer: i32,
}

#[repr(C)]
pub struct aicb_ctx {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct aicb_scene {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct aicb_group {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct aicb_group_scene {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct aicb_texture_target {
    _opaque: [u8; 0],
}
#[repr(C)]
pub struct aicb_group_texture_target {
    _opaque: [u8; 0],
}

/// `UpdateStrategy` of a texture target (all-is-cubes-gpu/src/raytrace_to_texture.rs:704-727, 835-918)
pub const AICB_TEXTURE_INCREMENTAL: c_int = 1;
pub const AICB_TEXTURE_CONSISTENT: c_int = 2;

/// a texture target's size, strategy, `dirty_pixels`, pick position and cycle length
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct aicb_texture_target_info {
    pub width: u32,
    pub height: u32,
    pub strategy: u32,
    pub _pad: u32,
    pub dirty_pixels: u64,
    pub next_pick: u64,
    pub cycle_length: u64,
}

/// one layer of `RtScene::trace_ray_through_layers` (renderer.rs:454-478)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_layer {
    pub scene: *mut aicb_scene,
    pub camera: *const aicb_camera,
    pub options: *const aicb_options,
}

/// one layer of a layered frame on a device group: a replicated scene
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_group_layer {
    pub scene: *mut aicb_group_scene,
    pub camera: *const aicb_camera,
    pub options: *const aicb_options,
}

/// every output in the caller's device memory: nullable device pointers of the call's device (device 0 on a group)
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct aicb_device_outputs {
    pub srgb8: *mut [u8; 4],
    pub rgba16f: *mut [u16; 4],
    pub colorbuf: *mut [f32; 4],
    pub depth: *mut f64,
    pub hit: *mut aicb_hit,
    pub steps: *mut u32,
    pub text: *mut i32,
    pub texel_rgba16f: *mut [u16; 4],
    pub texel_depth: *mut f32,
    pub terminal: *mut aicb_terminal_pixel,
    pub len: usize,
    pub full_frame: u32,
    pub _pad: u32,
}

unsafe extern "C" {
    pub fn aicb_abi_version() -> u32;
    pub fn aicb_ctx_create(device_id: c_int, out: *mut *mut aicb_ctx) -> aicb_status;
    pub fn aicb_ctx_destroy(ctx: *mut aicb_ctx);
    pub fn aicb_last_error() -> *const c_char;

    pub fn aicb_scene_create(ctx: *mut aicb_ctx, desc: *const aicb_scene_desc, out: *mut *mut aicb_scene) -> aicb_status;
    pub fn aicb_scene_update_cubes(s: *mut aicb_scene, cubes: *const [i32; 3], block_ids: *const u16, light: *const [u8; 4], n: usize) -> aicb_status;
    // SpaceChange::CubeBlock / CubeLight for every cube of a box: dense Z-major arrays, or one id (block_ids NULL)
    pub fn aicb_scene_update_region(s: *mut aicb_scene, region: *const aicb_aab, block_ids: *const u16, uniform_id: u16,
                                    light: *const [u8; 4]) -> aicb_status;
    pub fn aicb_scene_update_blocks(s: *mut aicb_scene, indices: *const u16, descs: *const aicb_block_desc, n: usize) -> aicb_status;
    // SpaceChange::BlockIndex for indices past the table: the blocks become the table's next indices
    pub fn aicb_scene_append_blocks(s: *mut aicb_scene, descs: *const aicb_block_desc, n: usize) -> aicb_status;
    // SpaceChange::EveryBlock: the table becomes [block] and every cube holds id 0; light is not touched
    pub fn aicb_scene_fill_uniform(s: *mut aicb_scene, block: *const aicb_block_desc) -> aicb_status;
    pub fn aicb_scene_upload_light(s: *mut aicb_scene, light: *const [u8; 4], n_texels: usize) -> aicb_status;
    pub fn aicb_scene_destroy(s: *mut aicb_scene);
    pub fn aicb_scene_device_bytes(s: *const aicb_scene) -> u64;
    pub fn aicb_scene_set_physics(s: *mut aicb_scene, sky: *const aicb_sky, light_max_distance: u8) -> aicb_status;
    // a scene fed from device memory: arrays in CUDA buffers of the scene's device, ordered on `stream` (a cudaStream_t,
    // NULL = the context's); validated on the device
    pub fn aicb_scene_update_cubes_device(s: *mut aicb_scene, d_cubes: *const [i32; 3], d_ids: *const u16,
                                          d_light_or_null: *const [u8; 4], n: usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_scene_update_region_device(s: *mut aicb_scene, region: *const aicb_aab, d_ids_or_null: *const u16,
                                           uniform_id: u16, d_light_or_null: *const [u8; 4],
                                           stream: *mut c_void) -> aicb_status;
    pub fn aicb_scene_upload_light_device(s: *mut aicb_scene, d_light: *const [u8; 4], n_texels: usize,
                                          stream: *mut c_void) -> aicb_status;
    pub fn aicb_scene_download_ids_device(s: *mut aicb_scene, d_out: *mut u16, n: usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_light_edit_cubes_device(s: *mut aicb_scene, d_cubes: *const [i32; 3], d_ids: *const u16, n: usize,
                                        n_changed_or_null: *mut usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_light_edit_region_device(s: *mut aicb_scene, region: *const aicb_aab, d_ids_or_null: *const u16,
                                         uniform_id: u16, n_changed_or_null: *mut usize,
                                         stream: *mut c_void) -> aicb_status;
    pub fn aicb_light_download_device(s: *mut aicb_scene, d_out: *mut [u8; 4], n_texels: usize,
                                      stream: *mut c_void) -> aicb_status;
    // descs[i].indices and descs[i].palette in the scene's device memory; `indices` and the descriptors on the host
    pub fn aicb_scene_update_blocks_device(s: *mut aicb_scene, indices: *const u16, descs: *const aicb_block_desc,
                                           n: usize, flags: u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_scene_append_blocks_device(s: *mut aicb_scene, descs: *const aicb_block_desc, n: usize, flags: u32,
                                           stream: *mut c_void) -> aicb_status;
    // the Space in the context's device memory: desc.block_ids, desc.light and every descriptor's indices and palette
    pub fn aicb_scene_create_device(ctx: *mut aicb_ctx, desc: *const aicb_scene_desc, flags: u32, stream: *mut c_void,
                                    out: *mut *mut aicb_scene) -> aicb_status;
    pub fn aicb_scene_fill_uniform_device(s: *mut aicb_scene, block: *const aicb_block_desc, flags: u32,
                                          stream: *mut c_void) -> aicb_status;

    pub fn aicb_shard_pixel_count(cam: *const aicb_camera, shard: *const aicb_shard) -> usize;
    pub fn aicb_render_srgb8(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, shard: *const aicb_shard,
                             out: *mut [u8; 4], out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_rgba16f(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, shard: *const aicb_shard,
                               out: *mut [u16; 4], out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_colorbuf(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, shard: *const aicb_shard,
                                out_colorbuf: *mut [f32; 4], depth: *mut f64, hit: *mut aicb_hit, steps: *mut u32,
                                out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_text(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, out: *mut i32, out_len: usize,
                            info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_layers_srgb8(world: *const aicb_layer, ui: *const aicb_layer, backdrop_rgba: *const [f32; 4],
                                    no_world_rgba: *const [f32; 4], out: *mut [u8; 4], out_len: usize,
                                    info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_layers_texture(world: *const aicb_layer, ui: *const aicb_layer, backdrop_rgba: *const [f32; 4],
                                      no_world_rgba: *const [f32; 4], depth_transform: *const [f64; 16],
                                      pixels: *const u32, n_pixels: usize, out_rgba16f: *mut [u16; 4],
                                      out_depth: *mut f32, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_layers_terminal(world: *const aicb_layer, ui: *const aicb_layer, backdrop_rgba: *const [f32; 4],
                                       no_world_rgba: *const [f32; 4], out: *mut aicb_terminal_pixel, out_len: usize,
                                       info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_ortho_image_size(s: *const aicb_scene, resolution: u32, width: *mut u32, height: *mut u32) -> aicb_status;
    pub fn aicb_render_orthographic(s: *mut aicb_scene, resolution: u32, out: *mut [u8; 4], out_len: usize,
                                    info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_srgb8_device(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, shard: *const aicb_shard,
                                    d_out: *mut c_void, out_len: usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_render_srgb8_device_frame(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                          shard: *const aicb_shard, d_frame: *mut c_void, frame_len: usize,
                                          stream: *mut c_void) -> aicb_status;
    pub fn aicb_render_finish(s: *mut aicb_scene, info: *mut aicb_render_info) -> aicb_status;
    // asynchronous, on `stream` (a cudaStream_t, NULL = the context's); aicb_render_finish completes them
    pub fn aicb_render_device(s: *mut aicb_scene, cam: *const aicb_camera, opt: *const aicb_options, shard: *const aicb_shard,
                              outs: *const aicb_device_outputs, stream: *mut c_void) -> aicb_status;
    pub fn aicb_render_views_srgb8(s: *mut aicb_scene, cameras: *const aicb_camera, n_views: usize,
                                   opt: *const aicb_options, out: *mut [u8; 4], out_len: usize,
                                   info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_views_rgba16f(s: *mut aicb_scene, cameras: *const aicb_camera, n_views: usize,
                                     opt: *const aicb_options, out: *mut [u16; 4], out_len: usize,
                                     info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_views_colorbuf(s: *mut aicb_scene, cameras: *const aicb_camera, n_views: usize,
                                      opt: *const aicb_options, out_colorbuf: *mut [f32; 4], depth: *mut f64,
                                      hit: *mut aicb_hit, steps: *mut u32, out_len: usize,
                                      info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_views_text(s: *mut aicb_scene, cameras: *const aicb_camera, n_views: usize,
                                  opt: *const aicb_options, out: *mut i32, out_len: usize,
                                  info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_render_views_device(s: *mut aicb_scene, d_cameras: *const aicb_camera, n_views: usize, fb_width: u32,
                                    fb_height: u32, opt: *const aicb_options, outs: *const aicb_device_outputs,
                                    stream: *mut c_void) -> aicb_status;
    pub fn aicb_trace_rays_device(s: *mut aicb_scene, d_origin_dir: *const [f64; 6], n: usize, opt: *const aicb_options,
                                  outs: *const aicb_device_outputs, stream: *mut c_void) -> aicb_status;
    pub fn aicb_render_layers_device(world: *const aicb_layer, ui: *const aicb_layer, backdrop_rgba: *const [f32; 4],
                                     no_world_rgba: *const [f32; 4], depth_transform: *const [f64; 16],
                                     d_pixels: *const u32, n_pixels: usize, outs: *const aicb_device_outputs,
                                     stream: *mut c_void) -> aicb_status;
    pub fn aicb_frame_create(ctx: *mut aicb_ctx, n_pixels: usize, d_frame: *mut *mut c_void, handle_out: *mut [u8; 64]) -> aicb_status;
    pub fn aicb_frame_open(ctx: *mut aicb_ctx, handle: *const [u8; 64], d_frame: *mut *mut c_void) -> aicb_status;
    pub fn aicb_frame_close(ctx: *mut aicb_ctx, d_frame: *mut c_void, opened: c_int) -> aicb_status;
    pub fn aicb_frame_read(ctx: *mut aicb_ctx, d_frame: *const c_void, out: *mut [u8; 4], n_pixels: usize, stream: *mut c_void) -> aicb_status;
    // delivery without a collective: two monotonic counters behind the frame's pixels (include/aicb200.h)
    pub fn aicb_frame_signal(ctx: *mut aicb_ctx, d_frame: *mut c_void, n_pixels: usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_frame_wait_arrived(ctx: *mut aicb_ctx, d_frame: *mut c_void, n_pixels: usize, count: u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_frame_release(ctx: *mut aicb_ctx, d_frame: *mut c_void, n_pixels: usize, frame_id: u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_frame_wait_consumed(ctx: *mut aicb_ctx, d_frame: *mut c_void, n_pixels: usize, frame_id: u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_frame_timed_out(ctx: *mut aicb_ctx, d_frame: *mut c_void, n_pixels: usize, out: *mut u32) -> aicb_status;
    pub fn aicb_ctx_stage_timing(ctx: *mut aicb_ctx, enable: c_int) -> aicb_status;
    pub fn aicb_ctx_device(ctx: *const aicb_ctx) -> c_int;
    // compute_derived's light fields of n blocks (blocking; writes `out` only on success)
    pub fn aicb_derive_block_light(ctx: *mut aicb_ctx, descs: *const aicb_block_desc, n: usize,
                                   out: *mut aicb_block_light) -> aicb_status;

    pub fn aicb_group_create(device_ids: *const c_int, n_devices: c_int, out: *mut *mut aicb_group) -> aicb_status;
    pub fn aicb_group_destroy(g: *mut aicb_group);
    pub fn aicb_group_size(g: *const aicb_group) -> c_int;
    pub fn aicb_group_scene_create(g: *mut aicb_group, desc: *const aicb_scene_desc, out: *mut *mut aicb_group_scene) -> aicb_status;
    pub fn aicb_group_scene_destroy(gs: *mut aicb_group_scene);
    pub fn aicb_group_scene_update_cubes(gs: *mut aicb_group_scene, cubes: *const [i32; 3], block_ids: *const u16,
                                         light: *const [u8; 4], n: usize) -> aicb_status;
    pub fn aicb_group_scene_update_region(gs: *mut aicb_group_scene, region: *const aicb_aab, block_ids: *const u16,
                                          uniform_id: u16, light: *const [u8; 4]) -> aicb_status;
    pub fn aicb_group_render_srgb8(gs: *mut aicb_group_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                   out: *mut [u8; 4], out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    // every replica; validated against replica 0 first, so a rejected call changes none
    pub fn aicb_group_scene_update_blocks(gs: *mut aicb_group_scene, indices: *const u16, descs: *const aicb_block_desc,
                                          n: usize) -> aicb_status;
    pub fn aicb_group_scene_upload_light(gs: *mut aicb_group_scene, light: *const [u8; 4], n_texels: usize) -> aicb_status;
    pub fn aicb_group_scene_set_physics(gs: *mut aicb_group_scene, sky: *const aicb_sky, light_max_distance: u8)
                                        -> aicb_status;
    // every replica; validated against replica 0 first, so a rejected call changes none
    pub fn aicb_group_scene_append_blocks(gs: *mut aicb_group_scene, descs: *const aicb_block_desc, n: usize) -> aicb_status;
    // every replica; validated once, so a rejected call changes none
    pub fn aicb_group_scene_fill_uniform(gs: *mut aicb_group_scene, block: *const aicb_block_desc) -> aicb_status;
    pub fn aicb_group_scene_update_cubes_device(gs: *mut aicb_group_scene, d_cubes: *const [i32; 3], d_ids: *const u16,
                                                d_light_or_null: *const [u8; 4], n: usize,
                                                stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_update_region_device(gs: *mut aicb_group_scene, region: *const aicb_aab,
                                                 d_ids_or_null: *const u16, uniform_id: u16,
                                                 d_light_or_null: *const [u8; 4], stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_upload_light_device(gs: *mut aicb_group_scene, d_light: *const [u8; 4], n_texels: usize,
                                                stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_download_ids_device(gs: *mut aicb_group_scene, d_out: *mut u16, n: usize,
                                                stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_light_edit_cubes_device(gs: *mut aicb_group_scene, d_cubes: *const [i32; 3], d_ids: *const u16,
                                              n: usize, n_changed_or_null: *mut usize,
                                              stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_light_edit_region_device(gs: *mut aicb_group_scene, region: *const aicb_aab,
                                               d_ids_or_null: *const u16, uniform_id: u16,
                                               n_changed_or_null: *mut usize, stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_light_download_device(gs: *mut aicb_group_scene, d_out: *mut [u8; 4], n_texels: usize,
                                            stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_update_blocks_device(gs: *mut aicb_group_scene, indices: *const u16,
                                                 descs: *const aicb_block_desc, n: usize, flags: u32,
                                                 stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_append_blocks_device(gs: *mut aicb_group_scene, descs: *const aicb_block_desc, n: usize,
                                                 flags: u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_scene_create_device(g: *mut aicb_group, desc: *const aicb_scene_desc, flags: u32,
                                          stream: *mut c_void, out: *mut *mut aicb_group_scene) -> aicb_status;
    pub fn aicb_group_scene_fill_uniform_device(gs: *mut aicb_group_scene, block: *const aicb_block_desc, flags: u32,
                                                stream: *mut c_void) -> aicb_status;
    // aicb_render_layers_* on a group: both layers must be scenes of the same group
    pub fn aicb_group_render_layers_srgb8(world: *const aicb_group_layer, ui: *const aicb_group_layer,
                                          backdrop_rgba: *const [f32; 4], no_world_rgba: *const [f32; 4],
                                          out: *mut [u8; 4], out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_layers_texture(world: *const aicb_group_layer, ui: *const aicb_group_layer,
                                            backdrop_rgba: *const [f32; 4], no_world_rgba: *const [f32; 4],
                                            depth_transform: *const [f64; 16], pixels: *const u32, n_pixels: usize,
                                            out_rgba16f: *mut [u16; 4], out_depth: *mut f32,
                                            info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_layers_terminal(world: *const aicb_group_layer, ui: *const aicb_group_layer,
                                             backdrop_rgba: *const [f32; 4], no_world_rgba: *const [f32; 4],
                                             out: *mut aicb_terminal_pixel, out_len: usize,
                                             info: *mut aicb_render_info) -> aicb_status;
    // the world-only single-context outputs on a group: whole frames, ray batches cut into warp ranges
    pub fn aicb_group_render_colorbuf(gs: *mut aicb_group_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                      out_colorbuf: *mut [f32; 4], depth: *mut f64, hit: *mut aicb_hit, steps: *mut u32,
                                      out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_rgba16f(gs: *mut aicb_group_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                     out: *mut [u16; 4], out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_trace_rays(gs: *mut aicb_group_scene, origin_dir: *const [f64; 6], n: usize,
                                 opt: *const aicb_options, out_colorbuf: *mut [f32; 4], depth: *mut f64,
                                 hit: *mut aicb_hit, steps: *mut u32, info: *mut aicb_render_info) -> aicb_status;
    // the device-output calls on a group: device-0 buffers, blocking; `stream` waits for the outputs
    pub fn aicb_group_render_device(gs: *mut aicb_group_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                    outs: *const aicb_device_outputs, stream: *mut c_void,
                                    info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_views_srgb8(gs: *mut aicb_group_scene, cameras: *const aicb_camera, n_views: usize,
                                         opt: *const aicb_options, out: *mut [u8; 4], out_len: usize,
                                         info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_views_rgba16f(gs: *mut aicb_group_scene, cameras: *const aicb_camera, n_views: usize,
                                           opt: *const aicb_options, out: *mut [u16; 4], out_len: usize,
                                           info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_views_colorbuf(gs: *mut aicb_group_scene, cameras: *const aicb_camera, n_views: usize,
                                            opt: *const aicb_options, out_colorbuf: *mut [f32; 4], depth: *mut f64,
                                            hit: *mut aicb_hit, steps: *mut u32, out_len: usize,
                                            info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_views_text(gs: *mut aicb_group_scene, cameras: *const aicb_camera, n_views: usize,
                                        opt: *const aicb_options, out: *mut i32, out_len: usize,
                                        info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_views_device(gs: *mut aicb_group_scene, d_cameras: *const aicb_camera, n_views: usize,
                                          fb_width: u32, fb_height: u32, opt: *const aicb_options,
                                          outs: *const aicb_device_outputs, stream: *mut c_void,
                                          info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_trace_rays_device(gs: *mut aicb_group_scene, d_origin_dir: *const [f64; 6], n: usize,
                                        opt: *const aicb_options, outs: *const aicb_device_outputs, stream: *mut c_void,
                                        info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_layers_device(world: *const aicb_group_layer, ui: *const aicb_group_layer,
                                           backdrop_rgba: *const [f32; 4], no_world_rgba: *const [f32; 4],
                                           depth_transform: *const [f64; 16], d_pixels: *const u32, n_pixels: usize,
                                           outs: *const aicb_device_outputs, stream: *mut c_void,
                                           info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_render_text(gs: *mut aicb_group_scene, cam: *const aicb_camera, opt: *const aicb_options,
                                  out: *mut i32, out_len: usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_ortho_image_size(gs: *const aicb_group_scene, resolution: u32, width: *mut u32, height: *mut u32)
                                       -> aicb_status;
    pub fn aicb_group_render_orthographic(gs: *mut aicb_group_scene, resolution: u32, out: *mut [u8; 4], out_len: usize,
                                          info: *mut aicb_render_info) -> aicb_status;

    // RaytraceToTexture's state on the device: the strategy, dirty_pixels and both render targets (blocking calls)
    pub fn aicb_texture_target_create(ctx: *mut aicb_ctx, width: u32, height: u32, strategy: c_int,
                                      out: *mut *mut aicb_texture_target) -> aicb_status;
    pub fn aicb_texture_target_destroy(t: *mut aicb_texture_target);
    pub fn aicb_texture_target_resize(t: *mut aicb_texture_target, width: u32, height: u32) -> aicb_status;
    pub fn aicb_texture_target_mark_dirty(t: *mut aicb_texture_target) -> aicb_status;
    pub fn aicb_texture_target_trace(t: *mut aicb_texture_target, world: *const aicb_layer, ui: *const aicb_layer,
                                     backdrop_rgba: *const [f32; 4], no_world_rgba: *const [f32; 4],
                                     depth_transform: *const [f64; 16], n: usize, n_traced: *mut usize,
                                     info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_texture_target_state(t: *const aicb_texture_target, out: *mut aicb_texture_target_info) -> aicb_status;
    pub fn aicb_texture_target_picks(t: *mut aicb_texture_target, start: u64, n: usize, out: *mut u32) -> aicb_status;
    pub fn aicb_texture_target_buffers(t: *mut aicb_texture_target, d_rgba16f: *mut *mut c_void,
                                       d_depth: *mut *mut c_void) -> aicb_status;
    pub fn aicb_texture_target_read(t: *mut aicb_texture_target, rgba16f: *mut [u16; 4], depth: *mut f32, n: usize)
                                    -> aicb_status;
    // the same on a device group: the targets are device 0's, a batch is cut into warp ranges across the devices
    pub fn aicb_group_texture_target_create(g: *mut aicb_group, width: u32, height: u32, strategy: c_int,
                                            out: *mut *mut aicb_group_texture_target) -> aicb_status;
    pub fn aicb_group_texture_target_destroy(t: *mut aicb_group_texture_target);
    pub fn aicb_group_texture_target_resize(t: *mut aicb_group_texture_target, width: u32, height: u32) -> aicb_status;
    pub fn aicb_group_texture_target_mark_dirty(t: *mut aicb_group_texture_target) -> aicb_status;
    pub fn aicb_group_texture_target_trace(t: *mut aicb_group_texture_target, world: *const aicb_group_layer,
                                           ui: *const aicb_group_layer, backdrop_rgba: *const [f32; 4],
                                           no_world_rgba: *const [f32; 4], depth_transform: *const [f64; 16], n: usize,
                                           n_traced: *mut usize, info: *mut aicb_render_info) -> aicb_status;
    pub fn aicb_group_texture_target_state(t: *const aicb_group_texture_target, out: *mut aicb_texture_target_info)
                                           -> aicb_status;
    pub fn aicb_group_texture_target_picks(t: *mut aicb_group_texture_target, start: u64, n: usize, out: *mut u32)
                                           -> aicb_status;
    pub fn aicb_group_texture_target_buffers(t: *mut aicb_group_texture_target, d_rgba16f: *mut *mut c_void,
                                             d_depth: *mut *mut c_void) -> aicb_status;
    pub fn aicb_group_texture_target_read(t: *mut aicb_group_texture_target, rgba16f: *mut [u16; 4], depth: *mut f32,
                                          n: usize) -> aicb_status;

    pub fn aicb_trace_rays(s: *mut aicb_scene, origin_dir: *const [f64; 6], n: usize, opt: *const aicb_options,
                           out_colorbuf: *mut [f32; 4], depth: *mut f64, hit: *mut aicb_hit, steps: *mut u32,
                           info: *mut aicb_render_info) -> aicb_status;

    pub fn aicb_camera_look_at(eye: *const [f64; 3], target: *const [f64; 3], fov_y_degrees: f64, view_distance: f64,
                               nominal_width: f64, nominal_height: f64, fb_width: u32, fb_height: u32, exposure: f32,
                               out: *mut aicb_camera) -> aicb_status;
    pub fn aicb_camera_from_view(rotation_ijkr: *const [f64; 4], translation: *const [f64; 3], fov_y_degrees: f64,
                                 view_distance: f64, nominal_width: f64, nominal_height: f64, fb_width: u32,
                                 fb_height: u32, exposure: f32, out: *mut aicb_camera) -> aicb_status;
    pub fn aicb_eye_for_look_at(bounds: *const aicb_aab, direction: *const [f64; 3], out_eye: *mut [f64; 3]);
    pub fn aicb_camera_project_ndc(cam: *const aicb_camera, ndc_x: f64, ndc_y: f64, out_origin_dir: *mut [f64; 6]);
    pub fn aicb_view_transform_matrix(rotation_ijkr: *const [f64; 4], translation: *const [f64; 3], out: *mut [f64; 16]);

    pub fn aicb_cursor_raycast(s: *mut aicb_scene, origin_dir: *const [f64; 6], max_distance_or_null: *const f64,
                               n: usize, out: *mut aicb_cursor) -> aicb_status;
    pub fn aicb_cursor_raycast_device(s: *mut aicb_scene, d_origin_dir: *const [f64; 6],
                                      d_max_distance_or_null: *const f64, n: usize, d_out: *mut aicb_cursor,
                                      stream: *mut c_void) -> aicb_status;
    pub fn aicb_project_cursor(world_or_null: *const aicb_layer, ui_or_null: *const aicb_layer, ndc: *const [f64; 2],
                               n: usize, world_max_distance: f64, out: *mut aicb_cursor) -> aicb_status;
    pub fn aicb_group_cursor_raycast(gs: *mut aicb_group_scene, origin_dir: *const [f64; 6],
                                     max_distance_or_null: *const f64, n: usize, out: *mut aicb_cursor)
                                     -> aicb_status;
    pub fn aicb_group_cursor_raycast_device(gs: *mut aicb_group_scene, d_origin_dir: *const [f64; 6],
                                            d_max_distance_or_null: *const f64, n: usize, d_out: *mut aicb_cursor,
                                            stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_project_cursor(world_or_null: *const aicb_group_layer, ui_or_null: *const aicb_group_layer,
                                     ndc: *const [f64; 2], n: usize, world_max_distance: f64, out: *mut aicb_cursor)
                                     -> aicb_status;

    pub fn aicb_step_bodies(s: *mut aicb_scene, bodies: *mut aicb_body, external_delta_v_or_null: *const [f64; 3],
                            n: usize, dt: f64, gravity: *const f64, info_or_null: *mut aicb_body_step_info,
                            contacts_or_null: *mut aicb_contact, max_contacts: u32) -> aicb_status;
    pub fn aicb_step_bodies_device(s: *mut aicb_scene, d_bodies: *mut aicb_body,
                                   d_external_delta_v_or_null: *const [f64; 3], n: usize, dt: f64,
                                   gravity: *const f64, d_info_or_null: *mut aicb_body_step_info,
                                   d_contacts_or_null: *mut aicb_contact, max_contacts: u32, stream: *mut c_void)
                                   -> aicb_status;
    pub fn aicb_group_step_bodies(gs: *mut aicb_group_scene, bodies: *mut aicb_body,
                                  external_delta_v_or_null: *const [f64; 3], n: usize, dt: f64, gravity: *const f64,
                                  info_or_null: *mut aicb_body_step_info, contacts_or_null: *mut aicb_contact,
                                  max_contacts: u32) -> aicb_status;
    pub fn aicb_group_step_bodies_device(gs: *mut aicb_group_scene, d_bodies: *mut aicb_body,
                                         d_external_delta_v_or_null: *const [f64; 3], n: usize, dt: f64,
                                         gravity: *const f64, d_info_or_null: *mut aicb_body_step_info,
                                         d_contacts_or_null: *mut aicb_contact, max_contacts: u32,
                                         stream: *mut c_void) -> aicb_status;

    pub fn aicb_step_exposure(s: *mut aicb_scene, states: *mut aicb_exposure_state, eye_to_world: *const [f64; 16],
                              n: usize, dt: f64, exposure_out_or_null: *mut f32) -> aicb_status;
    pub fn aicb_step_exposure_device(s: *mut aicb_scene, d_states: *mut aicb_exposure_state,
                                     d_eye_to_world: *const [f64; 16], n: usize, dt: f64,
                                     d_exposure_out_or_null: *mut f32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_step_exposure(gs: *mut aicb_group_scene, states: *mut aicb_exposure_state,
                                    eye_to_world: *const [f64; 16], n: usize, dt: f64, exposure_out_or_null: *mut f32)
                                    -> aicb_status;
    pub fn aicb_group_step_exposure_device(gs: *mut aicb_group_scene, d_states: *mut aicb_exposure_state,
                                           d_eye_to_world: *const [f64; 16], n: usize, dt: f64,
                                           d_exposure_out_or_null: *mut f32, stream: *mut c_void) -> aicb_status;

    pub fn aicb_look_rotation(yaw_degrees: f64, pitch_degrees: f64, out_ijkr: *mut [f64; 4]);
    pub fn aicb_step_eyes_device(s: *mut aicb_scene, d_eyes: *mut aicb_eye, d_bodies: *const aicb_body, n: usize,
                                 dt: f64, stream: *mut c_void) -> aicb_status;
    pub fn aicb_eye_views_device(s: *mut aicb_scene, d_eyes: *const aicb_eye, d_bodies: *const aicb_body,
                                 d_rotations: *const [f64; 4], d_exposures_or_null: *const f32, n: usize,
                                 params: *const aicb_eye_view_params, d_eye_to_world_or_null: *mut [f64; 16],
                                 d_cameras_or_null: *mut aicb_camera, d_look_rays_or_null: *mut [f64; 6],
                                 d_status_or_null: *mut u32, stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_step_eyes_device(gs: *mut aicb_group_scene, d_eyes: *mut aicb_eye, d_bodies: *const aicb_body,
                                       n: usize, dt: f64, stream: *mut c_void) -> aicb_status;
    pub fn aicb_group_eye_views_device(gs: *mut aicb_group_scene, d_eyes: *const aicb_eye,
                                       d_bodies: *const aicb_body, d_rotations: *const [f64; 4],
                                       d_exposures_or_null: *const f32, n: usize,
                                       params: *const aicb_eye_view_params,
                                       d_eye_to_world_or_null: *mut [f64; 16], d_cameras_or_null: *mut aicb_camera,
                                       d_look_rays_or_null: *mut [f64; 6], d_status_or_null: *mut u32,
                                       stream: *mut c_void) -> aicb_status;

    pub fn aicb_light_chart(weights: *mut f32, children: *mut u32) -> u32;
    pub fn aicb_light_chart_chains(preorder: *mut u32, chains: *mut [u32; 6], euler: *mut u16) -> u32;
    pub fn aicb_light_fast_evaluate(s: *mut aicb_scene) -> aicb_status;
    pub fn aicb_light_compute(s: *mut aicb_scene, cubes: *const [i32; 3], n: usize, out: *mut [u8; 4]) -> aicb_status;
    pub fn aicb_light_evaluate(s: *mut aicb_scene, epsilon: u8, updates_done: *mut u64, max_diff: *mut u8,
                               chart_node_visits: *mut u64) -> aicb_status;
    // LightStorage::update_light_from_queue with a budget of cube updates: the light step of a tick
    pub fn aicb_light_update_from_queue(s: *mut aicb_scene, max_updates: u64, info_or_null: *mut aicb_light_updates_info)
                                        -> aicb_status;
    // Mutation::set x n in list order, without propagation: a tick's SpaceChange::CubeBlock batch
    pub fn aicb_light_edit_cubes(s: *mut aicb_scene, cubes: *const [i32; 3], new_ids: *const u16, n: usize,
                                 n_changed_or_null: *mut usize) -> aicb_status;
    pub fn aicb_light_edit_and_propagate(s: *mut aicb_scene, cubes: *const [i32; 3], new_ids: *const u16, n_edits: usize,
                                         epsilon: u8, updates_done: *mut u64, max_diff: *mut u8) -> aicb_status;
    // Mutation::fill / fill_uniform(region): Mutation::set for every cube of a box, without propagation
    pub fn aicb_light_edit_region(s: *mut aicb_scene, region: *const aicb_aab, block_ids: *const u16, uniform_id: u16,
                                  n_changed_or_null: *mut usize) -> aicb_status;
    pub fn aicb_light_relight_blocks(s: *mut aicb_scene, indices: *const u16, n: usize, epsilon: u8, updates_done: *mut u64,
                                     max_diff: *mut u8) -> aicb_status;
    pub fn aicb_light_download(s: *mut aicb_scene, out: *mut [u8; 4], n_texels: usize) -> aicb_status;
    // the light update queue across save and load (all-is-cubes space.rs:290-313, save/conversion.rs:773-785)
    pub fn aicb_light_queue_uninitialized(s: *mut aicb_scene, n_queued_or_null: *mut usize) -> aicb_status;
    pub fn aicb_light_queue_region(s: *mut aicb_scene, region: *const aicb_aab, priority: u8) -> aicb_status;
    pub fn aicb_light_download_queue(s: *mut aicb_scene, priorities: *mut u8, n_texels: usize, n_queued_or_null: *mut usize)
                                     -> aicb_status;
    pub fn aicb_light_stats(s: *const aicb_scene, out: *mut [u64; 4]) -> aicb_status;
    pub fn aicb_light_changes_count(s: *const aicb_scene, n_changed: *mut usize) -> aicb_status;
    pub fn aicb_light_take_changes(s: *mut aicb_scene, indices: *mut u32, texels: *mut [u8; 4], capacity: usize,
                                   n_taken: *mut usize) -> aicb_status;
    // Space::compute_light::<LightUpdateCubeInfo>: aicb_light_compute's texels with each cube's rays
    pub fn aicb_light_compute_debug(s: *mut aicb_scene, cubes: *const [i32; 3], n: usize, out_texels: *mut [u8; 4],
                                    rays_or_null: *mut aicb_light_ray, ray_capacity: usize, ray_counts: *mut u32,
                                    n_rays_total: *mut usize) -> aicb_status;

    pub fn aicb_group_light_fast_evaluate(gs: *mut aicb_group_scene) -> aicb_status;
    pub fn aicb_group_light_compute(gs: *mut aicb_group_scene, cubes: *const [i32; 3], n: usize, out: *mut [u8; 4]) -> aicb_status;
    pub fn aicb_group_light_evaluate(gs: *mut aicb_group_scene, epsilon: u8, updates_done: *mut u64, max_diff: *mut u8,
                                     chart_node_visits: *mut u64) -> aicb_status;
    pub fn aicb_group_light_update_from_queue(gs: *mut aicb_group_scene, max_updates: u64,
                                              info_or_null: *mut aicb_light_updates_info) -> aicb_status;
    pub fn aicb_group_light_edit_and_propagate(gs: *mut aicb_group_scene, cubes: *const [i32; 3], new_ids: *const u16,
                                               n_edits: usize, epsilon: u8, updates_done: *mut u64, max_diff: *mut u8)
                                               -> aicb_status;
    pub fn aicb_group_light_edit_cubes(gs: *mut aicb_group_scene, cubes: *const [i32; 3], new_ids: *const u16, n: usize,
                                       n_changed_or_null: *mut usize) -> aicb_status;
    pub fn aicb_group_light_edit_region(gs: *mut aicb_group_scene, region: *const aicb_aab, block_ids: *const u16,
                                        uniform_id: u16, n_changed_or_null: *mut usize) -> aicb_status;
    pub fn aicb_group_light_relight_blocks(gs: *mut aicb_group_scene, indices: *const u16, n: usize, epsilon: u8,
                                           updates_done: *mut u64, max_diff: *mut u8) -> aicb_status;
    // the queue is device 0's; the scan reads replica 0's volume
    pub fn aicb_group_light_queue_uninitialized(gs: *mut aicb_group_scene, n_queued_or_null: *mut usize) -> aicb_status;
    pub fn aicb_group_light_queue_region(gs: *mut aicb_group_scene, region: *const aicb_aab, priority: u8) -> aicb_status;
    pub fn aicb_group_light_download_queue(gs: *mut aicb_group_scene, priorities: *mut u8, n_texels: usize,
                                           n_queued_or_null: *mut usize) -> aicb_status;
    pub fn aicb_group_light_download(gs: *mut aicb_group_scene, replica: c_int, out: *mut [u8; 4], n_texels: usize) -> aicb_status;
    pub fn aicb_group_light_stats(gs: *const aicb_group_scene, out: *mut [u64; 4]) -> aicb_status;
    pub fn aicb_group_light_changes_count(gs: *const aicb_group_scene, n_changed: *mut usize) -> aicb_status;
    pub fn aicb_group_light_take_changes(gs: *mut aicb_group_scene, indices: *mut u32, texels: *mut [u8; 4],
                                         capacity: usize, n_taken: *mut usize) -> aicb_status;
    pub fn aicb_group_light_compute_debug(gs: *mut aicb_group_scene, cubes: *const [i32; 3], n: usize,
                                          out_texels: *mut [u8; 4], rays_or_null: *mut aicb_light_ray, ray_capacity: usize,
                                          ray_counts: *mut u32, n_rays_total: *mut usize) -> aicb_status;
}
