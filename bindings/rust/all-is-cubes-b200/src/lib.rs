//! `B200Renderer`: the reference's `HeadlessRenderer` (all-is-cubes-render/src/headless.rs:17-44) on top of
//! `libaicb200` — a drop-in for `RtRenderer<()>` (raytracer/renderer.rs:38-355) wherever a
//! `Box<dyn HeadlessRenderer + Send>` is built (test-renderers/types/src/render.rs:61-82,
//! all-is-cubes-desktop/src/record.rs:210-236).
//!
//! * `update()` = `RtRenderer::update` (renderer.rs:96-161): camera sync, then per layer either a full snapshot
//!   (`SpaceRaytracer::new`, sr.rs:64-88 → `aicb_scene_create`) or the `SpaceChange` deltas an
//!   `UpdatingSpaceRaytracer` would apply (updating.rs:107-172 → `aicb_scene_append_blocks` / `_update_blocks` /
//!   `_update_cubes`).
//! * `draw()` = `RtRenderer::draw_rgba` (renderer.rs:282-308) with `trace_ray_through_layers` (renderer.rs:454-478)
//!   → `aicb_render_layers_srgb8`; the info text is drawn here over the returned pixels like renderer.rs:659-683.
//! * `trace_texture_batch()` = the tracing of `RaytraceToTexture::do_some_tracing` (raytrace_to_texture.rs:591-683)
//!   for a batch of pixels → `aicb_render_layers_texture`.
//! * `trace_texture_target()` = a whole `do_some_tracing` call on a `B200TextureTarget`: the pick order,
//!   `dirty_pixels` and both render targets stay on the device (`aicb_texture_target_trace`).
//! * `draw_terminal()` = the desktop terminal's `RtRenderer<CharacterRtData>::draw::<ColorCharacterBuf>`
//!   (all-is-cubes-desktop/src/terminal.rs:114-142, 341-394) → `aicb_render_layers_terminal`; the block indices it
//!   returns are mapped to `CharacterRtData` strings from one table per layer, kept current with the scenes.
//! * `B200Renderer::on_devices()` / `on_group()`: the same renderer on several devices (`aicb_group_*`): scenes
//!   replicated and kept current by the same deltas, `draw()` → `aicb_group_render_layers_srgb8`,
//!   `trace_texture_batch()` → `aicb_group_render_layers_texture`, `draw_terminal()` →
//!   `aicb_group_render_layers_terminal`.
//!
//! Not compiled in the repository this file ships in (no Rust toolchain there); see ../README.md.

mod convert;

use std::sync::{Arc, Mutex};

use all_is_cubes::character::Cursor;
use all_is_cubes::content::palette;
use all_is_cubes::listen::{self, Listen as _};
use all_is_cubes::math::{Cube, GridAab, Rgba, ZeroOne};
use all_is_cubes::space::{self, Space, SpaceChange};
use all_is_cubes::universe::{Handle, ReadTicket};
use all_is_cubes::util::maybe_sync::BoxFuture;
use all_is_cubes_b200_sys as sys;
use all_is_cubes_render::camera::{Camera, Layers, StandardCameras};
use all_is_cubes_render::{Flaws, HeadlessRenderer, RenderError, Rendering};

use unicode_segmentation::UnicodeSegmentation as _;

pub use convert::{block_desc_of, camera_of, options_of, sky_of, OwnedBlockDesc};

/// `aicb_status` other than OK, with the library's message (`aicb_last_error`).
#[derive(Clone, Debug)]
pub struct B200Error {
    pub status: sys::aicb_status,
    pub message: String,
}

fn check(status: sys::aicb_status) -> Result<(), B200Error> {
    if status == sys::AICB_OK {
        return Ok(());
    }
    // SAFETY: aicb_last_error never returns NULL; the string lives until the next failing call on this thread.
    let message = unsafe { std::ffi::CStr::from_ptr(sys::aicb_last_error()) }.to_string_lossy().into_owned();
    Err(B200Error { status, message })
}

/// One CUDA device + stream (`aicb_ctx`).  Shared by all renderers of a process.
#[derive(Debug)]
pub struct B200Context(*mut sys::aicb_ctx);
// SAFETY: the library serialises the calls on one context with its own mutex (include/aicb200.h, "Threading").
unsafe impl Send for B200Context {}
unsafe impl Sync for B200Context {}

impl B200Context {
    /// Fails with `AICB_ERR_CUDA` when there is no H100 (sm_90) GPU: there is no CPU fallback.
    pub fn new(device_id: i32) -> Result<Arc<Self>, B200Error> {
        let mut ctx = core::ptr::null_mut();
        check(unsafe { sys::aicb_ctx_create(device_id, &mut ctx) })?;
        Ok(Arc::new(Self(ctx)))
    }
}
impl Drop for B200Context {
    fn drop(&mut self) {
        unsafe { sys::aicb_ctx_destroy(self.0) }
    }
}

/// Several devices driven from this process (`aicb_group`): scenes replicated on each, frames cut into row strips,
/// texture batches into ranges of the pixel list, every device storing into device 0's buffers.
#[derive(Debug)]
pub struct B200Group(*mut sys::aicb_group);
// SAFETY: as B200Context: the library holds every context's lock for the whole of a group call.
unsafe impl Send for B200Group {}
unsafe impl Sync for B200Group {}

impl B200Group {
    /// `device_ids` may name a device more than once.  Fails if a device cannot reach device 0's memory (peer access).
    pub fn new(device_ids: &[i32]) -> Result<Arc<Self>, B200Error> {
        let mut group = core::ptr::null_mut();
        check(unsafe { sys::aicb_group_create(device_ids.as_ptr(), device_ids.len() as i32, &mut group) })?;
        Ok(Arc::new(Self(group)))
    }
}
impl Drop for B200Group {
    fn drop(&mut self) {
        unsafe { sys::aicb_group_destroy(self.0) }
    }
}

/// The depth transform of `RaytraceToTexture::do_some_tracing` (raytrace_to_texture.rs:613-618), composed by euclid
/// exactly as the reference composes it.
fn depth_transform_of(camera: &Camera) -> [f64; 16] {
    let depth_scale = -(camera.view_distance().into_inner() - camera.near_plane_distance().into_inner());
    let depth_bias = -camera.near_plane_distance().into_inner();
    camera
        .projection_matrix()
        .pre_translate(euclid::vec3(0., 0., depth_bias))
        .pre_scale(0., 0., depth_scale)
        .to_array()
}

#[derive(Clone, Copy, Debug)]
enum TargetHandle {
    Single(*mut sys::aicb_texture_target),
    Group(*mut sys::aicb_group_texture_target),
}

/// The state `RaytraceToTexture::Inner` keeps around its tracing (all-is-cubes-gpu/src/raytrace_to_texture.rs), on the
/// device (`aicb_texture_target_*`): the update strategy (`PixelPicker`'s order and position, or `Consistent`'s
/// `next`), `dirty_pixels`, and the `Rgba16Float` and `R32Float` render targets.  With it `do_some_tracing` becomes
/// `mark_dirty()` when `RtRenderer::update` reports a change, one `B200Renderer::trace_texture_target` per frame with
/// the caller's `rays_per_frame` rule, and an upload of the texels from `buffers()` (device memory) or `read()`.
#[derive(Debug)]
pub struct B200TextureTarget {
    handle: TargetHandle,
    _backend: Backend, // the context or group the target's buffers live on, kept alive as long as the target
}
// SAFETY: the library holds the target's context locks in every call.
unsafe impl Send for B200TextureTarget {}
unsafe impl Sync for B200TextureTarget {}

impl B200TextureTarget {
    fn new(backend: &Backend, width: u32, height: u32, incremental: bool) -> Result<Self, B200Error> {
        let strategy = if incremental { sys::AICB_TEXTURE_INCREMENTAL } else { sys::AICB_TEXTURE_CONSISTENT };
        let handle = match backend {
            Backend::Context(ctx) => {
                let mut t = core::ptr::null_mut();
                check(unsafe { sys::aicb_texture_target_create(ctx.0, width, height, strategy, &mut t) })?;
                TargetHandle::Single(t)
            }
            Backend::Group(g) => {
                let mut t = core::ptr::null_mut();
                check(unsafe { sys::aicb_group_texture_target_create(g.0, width, height, strategy, &mut t) })?;
                TargetHandle::Group(t)
            }
        };
        Ok(Self { handle, _backend: backend.clone() })
    }

    /// `UpdateStrategy::resize` and the textures' resize (:311-324): nothing for the same size.
    pub fn resize(&self, width: u32, height: u32) -> Result<(), B200Error> {
        check(match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_resize(t, width, height) },
            TargetHandle::Group(t) => unsafe { sys::aicb_group_texture_target_resize(t, width, height) },
        })
    }

    /// `RaytraceToTexture::dirty` (:587-589).
    pub fn mark_dirty(&self) -> Result<(), B200Error> {
        check(match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_mark_dirty(t) },
            TargetHandle::Group(t) => unsafe { sys::aicb_group_texture_target_mark_dirty(t) },
        })
    }

    pub fn state(&self) -> Result<sys::aicb_texture_target_info, B200Error> {
        let mut out = sys::aicb_texture_target_info::default();
        check(match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_state(t, &mut out) },
            TargetHandle::Group(t) => unsafe { sys::aicb_group_texture_target_state(t, &mut out) },
        })?;
        Ok(out)
    }

    /// The linear pixel indices of picks `start .. start + out.len()`: the texels a batch changed.
    pub fn picks(&self, start: u64, out: &mut [u32]) -> Result<(), B200Error> {
        check(match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_picks(t, start, out.len(), out.as_mut_ptr()) },
            TargetHandle::Group(t) => unsafe {
                sys::aicb_group_texture_target_picks(t, start, out.len(), out.as_mut_ptr())
            },
        })
    }

    /// Device pointers (the context's device, or the group's device 0) to the colour and depth texels, row-major;
    /// valid until the next `resize` or the target's drop.
    pub fn buffers(&self) -> Result<(*mut core::ffi::c_void, *mut core::ffi::c_void), B200Error> {
        let (mut color, mut depth) = (core::ptr::null_mut(), core::ptr::null_mut());
        check(match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_buffers(t, &mut color, &mut depth) },
            TargetHandle::Group(t) => unsafe { sys::aicb_group_texture_target_buffers(t, &mut color, &mut depth) },
        })?;
        Ok((color, depth))
    }

    /// Copies of both render targets (`width * height` texels each, row-major).
    pub fn read(&self, color: &mut [[u16; 4]], depth: &mut [f32]) -> Result<(), B200Error> {
        assert_eq!(color.len(), depth.len(), "one depth texel per colour texel");
        check(match self.handle {
            TargetHandle::Single(t) => unsafe {
                sys::aicb_texture_target_read(t, color.as_mut_ptr(), depth.as_mut_ptr(), color.len())
            },
            TargetHandle::Group(t) => unsafe {
                sys::aicb_group_texture_target_read(t, color.as_mut_ptr(), depth.as_mut_ptr(), color.len())
            },
        })
    }
}
impl Drop for B200TextureTarget {
    fn drop(&mut self) {
        match self.handle {
            TargetHandle::Single(t) => unsafe { sys::aicb_texture_target_destroy(t) },
            TargetHandle::Group(t) => unsafe { sys::aicb_group_texture_target_destroy(t) },
        }
    }
}

/// Where a renderer's scenes live.
#[derive(Clone, Debug)]
enum Backend {
    Context(Arc<B200Context>),
    Group(Arc<B200Group>),
}

/// One layer's device-resident scene: on one context, or replicated on a group.
#[derive(Clone, Copy, Debug)]
enum SceneHandle {
    Single(*mut sys::aicb_scene),
    Group(*mut sys::aicb_group_scene),
}

impl SceneHandle {
    fn create(backend: &Backend, desc: &sys::aicb_scene_desc) -> Result<Self, B200Error> {
        match backend {
            Backend::Context(ctx) => {
                let mut s = core::ptr::null_mut();
                check(unsafe { sys::aicb_scene_create(ctx.0, desc, &mut s) })?;
                Ok(Self::Single(s))
            }
            Backend::Group(group) => {
                let mut s = core::ptr::null_mut();
                check(unsafe { sys::aicb_group_scene_create(group.0, desc, &mut s) })?;
                Ok(Self::Group(s))
            }
        }
    }

    fn update_blocks(self, indices: &[u16], descs: &[sys::aicb_block_desc]) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_scene_update_blocks(s, indices.as_ptr(), descs.as_ptr(), indices.len()),
                Self::Group(s) => sys::aicb_group_scene_update_blocks(s, indices.as_ptr(), descs.as_ptr(), indices.len()),
            }
        })
    }

    fn append_blocks(self, descs: &[sys::aicb_block_desc]) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_scene_append_blocks(s, descs.as_ptr(), descs.len()),
                Self::Group(s) => sys::aicb_group_scene_append_blocks(s, descs.as_ptr(), descs.len()),
            }
        })
    }

    fn fill_uniform(self, block: &sys::aicb_block_desc) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_scene_fill_uniform(s, block),
                Self::Group(s) => sys::aicb_group_scene_fill_uniform(s, block),
            }
        })
    }

    fn light_queue_region(self, region: &sys::aicb_aab, priority: u8) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_light_queue_region(s, region, priority),
                Self::Group(s) => sys::aicb_group_light_queue_region(s, region, priority),
            }
        })
    }

    fn update_cubes(self, cubes: &[[i32; 3]], ids: &[u16], light: &[[u8; 4]]) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_scene_update_cubes(s, cubes.as_ptr(), ids.as_ptr(), light.as_ptr(), cubes.len()),
                Self::Group(s) => {
                    sys::aicb_group_scene_update_cubes(s, cubes.as_ptr(), ids.as_ptr(), light.as_ptr(), cubes.len())
                }
            }
        })
    }

    fn update_region(self, region: &sys::aicb_aab, fill: RegionFill<'_>, light: Option<&[[u8; 4]]>) -> Result<(), B200Error> {
        let (ids, uniform) = fill.as_ffi();
        let light = light.map_or(core::ptr::null(), <[[u8; 4]]>::as_ptr);
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_scene_update_region(s, region, ids, uniform, light),
                Self::Group(s) => sys::aicb_group_scene_update_region(s, region, ids, uniform, light),
            }
        })
    }

    fn light_edit_region(self, region: &sys::aicb_aab, fill: RegionFill<'_>) -> Result<usize, B200Error> {
        let (ids, uniform) = fill.as_ffi();
        let mut changed = 0usize;
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_light_edit_region(s, region, ids, uniform, &mut changed),
                Self::Group(s) => sys::aicb_group_light_edit_region(s, region, ids, uniform, &mut changed),
            }
        })?;
        Ok(changed)
    }

    fn light_edit_cubes(self, cubes: &[[i32; 3]], ids: &[u16]) -> Result<usize, B200Error> {
        let mut changed = 0usize;
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_light_edit_cubes(s, cubes.as_ptr(), ids.as_ptr(), cubes.len(), &mut changed),
                Self::Group(s) => sys::aicb_group_light_edit_cubes(s, cubes.as_ptr(), ids.as_ptr(), cubes.len(), &mut changed),
            }
        })?;
        Ok(changed)
    }

    fn step_exposure(self, states: &mut [sys::aicb_exposure_state], eye_to_world: &[[f64; 16]], dt: f64,
                     exposures: &mut [f32]) -> Result<(), B200Error> {
        check(unsafe {
            match self {
                Self::Single(s) => sys::aicb_step_exposure(s, states.as_mut_ptr(), eye_to_world.as_ptr(), states.len(),
                                                           dt, exposures.as_mut_ptr()),
                Self::Group(s) => sys::aicb_group_step_exposure(s, states.as_mut_ptr(), eye_to_world.as_ptr(),
                                                                states.len(), dt, exposures.as_mut_ptr()),
            }
        })
    }

    fn destroy(self) {
        match self {
            Self::Single(s) => unsafe { sys::aicb_scene_destroy(s) },
            Self::Group(s) => unsafe { sys::aicb_group_scene_destroy(s) },
        }
    }

    // A renderer's scenes all live on its backend.
    fn single(self) -> *mut sys::aicb_scene {
        match self {
            Self::Single(s) => s,
            Self::Group(_) => unreachable!("a group scene on a single-context renderer"),
        }
    }
    fn grouped(self) -> *mut sys::aicb_group_scene {
        match self {
            Self::Group(s) => s,
            Self::Single(_) => unreachable!("a single-context scene on a group renderer"),
        }
    }
}

/// What a box of cubes is filled with: one block index, or one per cube, Z-major within the box (`Vol`'s order).
#[derive(Clone, Copy, Debug)]
pub enum RegionFill<'a> {
    Uniform(space::BlockIndex),
    Each(&'a [space::BlockIndex]),
}
impl RegionFill<'_> {
    fn as_ffi(self) -> (*const u16, u16) {
        match self {
            Self::Uniform(id) => (core::ptr::null(), id),
            Self::Each(ids) => (ids.as_ptr(), 0),
        }
    }
    fn fits(self, region: GridAab) -> bool {
        match self {
            Self::Uniform(_) => true,
            Self::Each(ids) => ids.len() == region.volume().unwrap_or(usize::MAX),
        }
    }
}

/// The `SpaceChange` buckets of `SrtTodo` (updating.rs:176-219).
#[derive(Debug, Default)]
struct Todo {
    listener: bool,
    everything: bool,
    blocks: std::collections::HashSet<space::BlockIndex>,
    cubes: std::collections::HashSet<Cube>,
}
impl listen::Store<SpaceChange> for Todo {
    fn receive(&mut self, messages: &[SpaceChange]) {
        for message in messages {
            match *message {
                SpaceChange::EveryBlock => {
                    self.everything = true;
                    self.blocks.clear();
                    self.cubes.clear();
                }
                SpaceChange::CubeLight { cube, .. } | SpaceChange::CubeBlock { cube, .. } => {
                    self.cubes.insert(cube);
                }
                SpaceChange::BlockIndex(index) | SpaceChange::BlockEvaluation(index) => {
                    self.blocks.insert(index);
                }
                SpaceChange::Physics => {}
            }
        }
    }
}

/// Device-resident copy of one `Space` kept current from its change notifications:
/// the counterpart of `UpdatingSpaceRaytracer` (updating.rs:19-172).
struct SceneFollower {
    space: Handle<Space>,
    scene: Option<SceneHandle>,
    todo: listen::StoreLock<Todo>,
    /// `CharacterRtData` of every block index (the terminal's text), current with `scene`
    chars: Vec<String>,
}

/// `CharacterRtData::from_block` (raytracer/text.rs:30-38): the first grapheme of the block's display name, or "#".
fn character_of(data: &space::SpaceBlockData) -> String {
    let name: &str = &data.evaluated().attributes().display_name;
    name.graphemes(true).next().unwrap_or("#").to_owned()
}
// SAFETY: see B200Context.
unsafe impl Send for SceneFollower {}

impl SceneFollower {
    fn new(space: Handle<Space>) -> Self {
        Self {
            space,
            scene: None,
            todo: listen::StoreLock::new(Todo { listener: true, everything: true, ..Todo::default() }),
            chars: Vec::new(),
        }
    }

    fn update(&mut self, backend: &Backend, read_ticket: ReadTicket<'_>) -> Result<bool, RenderError> {
        let todo = {
            let mut guard = self.todo.lock();
            if !guard.listener && !guard.everything && guard.blocks.is_empty() && guard.cubes.is_empty() {
                return Ok(false);
            }
            core::mem::take(&mut *guard)
        };
        let space = self.space.read(read_ticket).map_err(RenderError::Read)?;
        if todo.listener {
            space.listen(self.todo.listener());
        }
        if self.scene.is_none() {
            // SpaceRaytracer::new (sr.rs:64-88): bounds, extract() of (block index, light texel), block_data(), sky
            let bounds = space.bounds();
            let cubes = space.extract(bounds, |e| (e.block_index(), e.light().as_texel())); // space.rs:740-761, Z-major
            let ids: Vec<u16> = cubes.as_linear().iter().map(|c| c.0).collect();
            let light: Vec<[u8; 4]> = cubes.as_linear().iter().map(|c| c.1).collect();
            let owned: Vec<OwnedBlockDesc> = space.block_data().iter().map(block_desc_of).collect();
            let blocks: Vec<sys::aicb_block_desc> = owned.iter().map(OwnedBlockDesc::as_ffi).collect();
            let physics = space.physics();
            let desc = sys::aicb_scene_desc {
                bounds: convert::aab_of(bounds),
                block_ids: ids.as_ptr(),
                // LightPhysics::None => PackedLight::ONE everywhere (space.rs:1241-1246): no light volume
                light: if matches!(physics.light, space::LightPhysics::None) { core::ptr::null() } else { light.as_ptr() },
                blocks: blocks.as_ptr(),
                n_blocks: blocks.len(),
                sky: sky_of(&physics.sky),
                light_max_distance: convert::light_max_distance_of(&physics.light),
                _pad: [0; 7],
            };
            let fresh = SceneHandle::create(backend, &desc).map_err(to_render_error)?;
            if let Some(old) = self.scene.replace(fresh) {
                old.destroy();
            }
            self.chars = space.block_data().iter().map(character_of).collect();
        } else if let Some(scene) = self.scene {
            // SpaceChange::EveryBlock: Mutation::fill_uniform over the whole bounds (space.rs:1461-1474), the one
            // source of it, left every cube holding palette index 0.  The scene takes the fill in place (the table
            // becomes [data[0]]) and, if the Space is lit, queues every cube at Priority::UNINIT as the reference
            // does; the light texels stay as they are.  The changes that came after it follow below.
            if todo.everything {
                let data = space.block_data();
                let block = block_desc_of(&data[0]);
                scene.fill_uniform(&block.as_ffi()).map_err(to_render_error)?;
                if !matches!(space.physics().light, space::LightPhysics::None) {
                    scene.light_queue_region(&convert::aab_of(space.bounds()), 210).map_err(to_render_error)?;
                }
                self.chars = vec![character_of(&data[0])];
            }
            // SpaceChange::BlockIndex for indices past the table: append TracingBlock::from_block of every entry the
            // scene lacks (updating.rs:145-151); on a group every replica takes them (aicb_group_scene_append_blocks)
            let known = self.chars.len();
            let data = space.block_data();
            if data.len() > known {
                let owned: Vec<OwnedBlockDesc> = data[known..].iter().map(block_desc_of).collect();
                let descs: Vec<sys::aicb_block_desc> = owned.iter().map(OwnedBlockDesc::as_ffi).collect();
                scene.append_blocks(&descs).map_err(to_render_error)?;
                self.chars.extend(data[known..].iter().map(character_of));
            }
            // SpaceChange::BlockIndex / BlockEvaluation of indices the scene already had: re-run
            // TracingBlock::from_block for those (updating.rs:152-157); on a group every replica takes them
            // (aicb_group_scene_update_blocks), no rebuild
            let idx: Vec<u16> = todo.blocks.iter().copied().filter(|&i| usize::from(i) < known).collect();
            if !idx.is_empty() {
                let owned: Vec<OwnedBlockDesc> = idx.iter().map(|&i| block_desc_of(&data[usize::from(i)])).collect();
                let descs: Vec<sys::aicb_block_desc> = owned.iter().map(OwnedBlockDesc::as_ffi).collect();
                scene.update_blocks(&idx, &descs).map_err(to_render_error)?;
                for &i in &idx {
                    self.chars[usize::from(i)] = character_of(&data[usize::from(i)]);
                }
            }
            // SpaceChange::CubeBlock / CubeLight (updating.rs:151-166)
            if !todo.cubes.is_empty() {
                let mut cubes = Vec::with_capacity(todo.cubes.len());
                let mut ids = Vec::with_capacity(todo.cubes.len());
                let mut light = Vec::with_capacity(todo.cubes.len());
                for &cube in &todo.cubes {
                    if let Some(index) = space.get_block_index(cube) {
                        cubes.push([cube.x, cube.y, cube.z]);
                        ids.push(index);
                        light.push(space.get_lighting(cube).as_texel());
                    }
                }
                scene.update_cubes(&cubes, &ids, &light).map_err(to_render_error)?;
            }
        }
        Ok(true)
    }
}
impl Drop for SceneFollower {
    fn drop(&mut self) {
        if let Some(scene) = self.scene.take() {
            scene.destroy();
        }
    }
}

fn to_render_error(e: B200Error) -> RenderError {
    // The reference has no variant for "lost GPU / out of memory" yet (lib.rs:46-58, "TODO: add errors for out of
    // memory, lost GPU"); RenderError::Read is its only one.  Until it grows one, surface the message and abort the
    // frame like a panic in RtRenderer would (renderer.rs:193-197 panics on a size mismatch).
    panic!("libaicb200: status {} — {}", e.status, e.message)
}

/// Drop-in for `RtRenderer<()>`.
pub struct B200Renderer {
    backend: Backend,
    cameras: StandardCameras,
    layers: Layers<Option<SceneFollower>>,
    had_cursor: bool,
}

impl B200Renderer {
    /// == `RtRenderer::new(cameras, size_policy = identity, custom_options = ())` (renderer.rs:65-81)
    pub fn new(ctx: Arc<B200Context>, cameras: StandardCameras) -> Self {
        Self::with_backend(Backend::Context(ctx), cameras)
    }

    /// The same renderer on a device group: each layer's Space is replicated on every device, kept current by the
    /// same deltas, and every frame or texture batch is shared between the devices (`aicb_group_render_layers_*`).
    /// The pixels are those `new` draws, bit for bit.
    pub fn on_group(group: Arc<B200Group>, cameras: StandardCameras) -> Self {
        Self::with_backend(Backend::Group(group), cameras)
    }

    /// `on_group` with a group of its own over `device_ids`.
    pub fn on_devices(device_ids: &[i32], cameras: StandardCameras) -> Result<Self, B200Error> {
        Ok(Self::on_group(B200Group::new(device_ids)?, cameras))
    }

    fn with_backend(backend: Backend, cameras: StandardCameras) -> Self {
        Self { backend, cameras, layers: Layers { world: None, ui: None }, had_cursor: false }
    }

    /// The world layer's scene, once `update()` has created it.
    fn world_scene(&self) -> Result<SceneHandle, B200Error> {
        self.layers.world.as_ref().and_then(|f| f.scene).ok_or_else(|| B200Error {
            status: sys::AICB_ERR_INVALID,
            message: "no world scene yet: call update() first".into(),
        })
    }

    /// For a host that fills a box of the world Space itself (`Space::fill`, `fill_uniform` over a region,
    /// `SpaceTransaction::filling`) and sends the box instead of waiting for one `SpaceChange::CubeBlock` per cube:
    /// the box's new block indices, and its light texels if given, Z-major within `region`
    /// (`aicb_scene_update_region`).  The follower still applies the per-cube changes the Space announces, to the
    /// same values.
    pub fn update_world_region(&self, region: GridAab, fill: RegionFill<'_>, light: Option<&[[u8; 4]]>) -> Result<(), B200Error> {
        assert!(fill.fits(region) && light.map_or(true, |l| l.len() == region.volume().unwrap_or(usize::MAX)),
                "array length is not the region's volume");
        self.world_scene()?.update_region(&convert::aab_of(region), fill, light)
    }

    /// The same fill on a world scene whose light the library computes: `Mutation::set`'s light rule for every cube of
    /// `region` whose block changes, on the device (`aicb_light_edit_region`).  Returns the number of changed cubes;
    /// nothing propagates until the host asks for it (`aicb_light_evaluate`).
    pub fn light_edit_world_region(&self, region: GridAab, fill: RegionFill<'_>) -> Result<usize, B200Error> {
        assert!(fill.fits(region), "array length is not the region's volume");
        self.world_scene()?.light_edit_region(&convert::aab_of(region), fill)
    }

    /// A tick's scattered `Mutation::set`s on a world scene whose light the library computes: `cubes[i]` takes block
    /// index `ids[i]`, in list order, with `Mutation::set`'s light rule on the device and no propagation
    /// (`aicb_light_edit_cubes`).  A cube may be named more than once.  Returns the number of entries that changed a
    /// block, the `SpaceChange::CubeBlock`s the Space sends for the list; the light moves when the host asks for it
    /// (`aicb_light_update_from_queue`).
    pub fn light_edit_world_cubes(&self, cubes: &[Cube], ids: &[u16]) -> Result<usize, B200Error> {
        assert_eq!(cubes.len(), ids.len(), "one block index per cube");
        let cubes: Vec<[i32; 3]> = cubes.iter().map(|c| [c.x, c.y, c.z]).collect();
        self.world_scene()?.light_edit_cubes(&cubes, ids)
    }

    /// `character::exposure::State::step` (character/exposure.rs:67-136) for a world that lives on the GPU, where no
    /// reference `Character` steps its own exposure: each of `states` by one tick of `dt` seconds against the world
    /// scene, from the eye whose view transform is `eye_to_world[i]` (`convert::view_transform_of`);
    /// `exposures[i]` receives `State::exposure()`, which the host hands to `Camera::set_measured_exposure`
    /// (`aicb_step_exposure`).  A Space kept in Rust needs none of this: `StandardCameras` applies its character's own.
    pub fn step_world_exposure(&self, states: &mut [sys::aicb_exposure_state], eye_to_world: &[[f64; 16]], dt: f64,
                               exposures: &mut [f32]) -> Result<(), B200Error> {
        assert!(eye_to_world.len() == states.len() && exposures.len() == states.len(), "one matrix and one exposure per state");
        self.world_scene()?.step_exposure(states, eye_to_world, dt, exposures)
    }

    /// Calls `single` with the layers this renderer holds as `aicb_layer`s, or on a group `group` with them as
    /// `aicb_group_layer`s (NULL for an absent layer).
    fn with_layers<R>(
        &self,
        cams: &Layers<Camera>,
        single: impl FnOnce(*const sys::aicb_layer, *const sys::aicb_layer) -> R,
        group: impl FnOnce(*const sys::aicb_group_layer, *const sys::aicb_group_layer) -> R,
    ) -> R {
        let world_cam = camera_of(&cams.world);
        let world_opt = options_of(cams.world.options());
        let ui_cam = camera_of(&cams.ui);
        let ui_opt = options_of(cams.ui.options());
        let w = self.layers.world.as_ref().and_then(|f| f.scene);
        let u = self.layers.ui.as_ref().and_then(|f| f.scene);
        match self.backend {
            Backend::Context(_) => {
                let world = w.map(|s| sys::aicb_layer { scene: s.single(), camera: &world_cam, options: &world_opt });
                let ui = u.map(|s| sys::aicb_layer { scene: s.single(), camera: &ui_cam, options: &ui_opt });
                single(world.as_ref().map_or(core::ptr::null(), |l| l), ui.as_ref().map_or(core::ptr::null(), |l| l))
            }
            Backend::Group(_) => {
                let world = w.map(|s| sys::aicb_group_layer { scene: s.grouped(), camera: &world_cam, options: &world_opt });
                let ui = u.map(|s| sys::aicb_group_layer { scene: s.grouped(), camera: &ui_cam, options: &ui_opt });
                group(world.as_ref().map_or(core::ptr::null(), |l| l), ui.as_ref().map_or(core::ptr::null(), |l| l))
            }
        }
    }

    /// The body of `RaytraceToTexture::do_some_tracing` (all-is-cubes-gpu/src/raytrace_to_texture.rs:591-683) for one
    /// batch: `trace_one` for each pixel of `pixels` (linear indices `y * width + x`, e.g. what `PixelPicker` yields;
    /// `None` = the whole texture, row-major), through the layers this renderer holds, on the GPU.  `cams` are the
    /// cameras of the caller's `RtScene` (with its size policy applied).  `color[i]` receives the `Rgba16Float` texel
    /// as raw f16 bits and `depth[i]` the `R32Float` texel of the i-th pixel; the caller stores them with
    /// `set_pixel` as `store_one` does.
    pub fn trace_texture_batch(
        &self,
        cams: &Layers<Camera>,
        pixels: Option<&[u32]>,
        color: &mut [[u16; 4]],
        depth: &mut [f32],
    ) -> Result<sys::aicb_render_info, B200Error> {
        let depth_transform = depth_transform_of(&cams.world);

        let backdrop: Rgba = self.cameras.ui_view_state().backdrop;
        let backdrop_arr: [f32; 4] = backdrop.into();
        let backdrop_ptr: *const [f32; 4] = if backdrop == Rgba::TRANSPARENT { core::ptr::null() } else { &backdrop_arr };
        let no_world: [f32; 4] = palette::NO_WORLD_TO_SHOW.into();
        let n = pixels.map_or(color.len(), <[u32]>::len);
        assert!(color.len() >= n && depth.len() >= n, "output slices shorter than the batch");
        let list = pixels.map_or(core::ptr::null(), <[u32]>::as_ptr);
        let (color, depth) = (color.as_mut_ptr(), depth.as_mut_ptr());

        let mut info = sys::aicb_render_info::default();
        let info_ptr: *mut sys::aicb_render_info = &mut info;
        check(self.with_layers(
            cams,
            |world, ui| unsafe {
                sys::aicb_render_layers_texture(world, ui, backdrop_ptr, &no_world, &depth_transform, list, n, color, depth,
                                                info_ptr)
            },
            |world, ui| unsafe {
                sys::aicb_group_render_layers_texture(world, ui, backdrop_ptr, &no_world, &depth_transform, list, n, color,
                                                      depth, info_ptr)
            },
        ))?;
        Ok(info)
    }

    /// One `RaytraceToTexture::do_some_tracing` batch into a `B200TextureTarget` of this renderer's backend:
    /// `rays_per_frame` picks from the target's update strategy, traced through the layers this renderer holds and
    /// stored into the target's render targets on the device (`aicb_texture_target_trace`).  Returns the picks traced
    /// (0 once `dirty_pixels` is 0) and the batch's info; the caller times the call for its `rays_per_frame` rule.
    pub fn trace_texture_target(
        &self,
        target: &B200TextureTarget,
        cams: &Layers<Camera>,
        rays_per_frame: usize,
    ) -> Result<(usize, sys::aicb_render_info), B200Error> {
        let depth_transform = depth_transform_of(&cams.world);
        let backdrop: Rgba = self.cameras.ui_view_state().backdrop;
        let backdrop_arr: [f32; 4] = backdrop.into();
        let backdrop_ptr: *const [f32; 4] = if backdrop == Rgba::TRANSPARENT { core::ptr::null() } else { &backdrop_arr };
        let no_world: [f32; 4] = palette::NO_WORLD_TO_SHOW.into();
        let mut info = sys::aicb_render_info::default();
        let info_ptr: *mut sys::aicb_render_info = &mut info;
        let mut traced = 0usize;
        let traced_ptr: *mut usize = &mut traced;
        check(self.with_layers(
            cams,
            |world, ui| match target.handle {
                TargetHandle::Single(t) => unsafe {
                    sys::aicb_texture_target_trace(t, world, ui, backdrop_ptr, &no_world, &depth_transform,
                                                   rays_per_frame, traced_ptr, info_ptr)
                },
                TargetHandle::Group(_) => sys::AICB_ERR_INVALID,
            },
            |world, ui| match target.handle {
                TargetHandle::Group(t) => unsafe {
                    sys::aicb_group_texture_target_trace(t, world, ui, backdrop_ptr, &no_world, &depth_transform,
                                                         rays_per_frame, traced_ptr, info_ptr)
                },
                TargetHandle::Single(_) => sys::AICB_ERR_INVALID,
            },
        ))?;
        Ok((traced, info))
    }

    /// A `B200TextureTarget` on this renderer's context or group.
    pub fn texture_target(&self, width: u32, height: u32, incremental: bool) -> Result<B200TextureTarget, B200Error> {
        B200TextureTarget::new(&self.backend, width, height, incremental)
    }

    /// The desktop terminal's frame (all-is-cubes-desktop/src/terminal.rs:114-142), in place of
    /// `scene.draw::<ColorCharacterBuf, _, _, _>(|_| String::new(), |b| b.output(camera), &mut image)`: per pixel of
    /// the world camera's framebuffer, row-major, the `CharacterBuf` string and
    /// `Some(camera.post_process_color(Rgba::from(ColorBuf)))` (ColorCharacterBuf::output, :355-366), through the
    /// layers this renderer holds, and the image's info.  The info text is empty, as the terminal draws it.
    pub fn draw_terminal(&self) -> Result<(Vec<(String, Option<Rgba>)>, sys::aicb_render_info), B200Error> {
        let cams: &Layers<Camera> = self.cameras.cameras();
        let size = cams.world.viewport().framebuffer_size;
        let mut pixels = vec![sys::aicb_terminal_pixel::default(); (size.width as usize) * (size.height as usize)];
        let backdrop: Rgba = self.cameras.ui_view_state().backdrop;
        let backdrop_arr: [f32; 4] = backdrop.into();
        let backdrop_ptr: *const [f32; 4] = if backdrop == Rgba::TRANSPARENT { core::ptr::null() } else { &backdrop_arr };
        let no_world: [f32; 4] = palette::NO_WORLD_TO_SHOW.into();
        let mut info = sys::aicb_render_info::default();
        if self.layers.world.is_none() && self.layers.ui.is_none() {
            // no Space at all: every accumulator is P::paint(NO_WORLD_TO_SHOW) (renderer.rs:474-477)
            let c = cams.world.post_process_color(palette::NO_WORLD_TO_SHOW);
            return Ok((vec![(" ".to_owned(), Some(c)); pixels.len()], info));
        }
        let (out, out_len) = (pixels.as_mut_ptr(), pixels.len());
        let info_ptr: *mut sys::aicb_render_info = &mut info;
        check(self.with_layers(
            cams,
            |world, ui| unsafe {
                sys::aicb_render_layers_terminal(world, ui, backdrop_ptr, &no_world, out, out_len, info_ptr)
            },
            |world, ui| unsafe {
                sys::aicb_group_render_layers_terminal(world, ui, backdrop_ptr, &no_world, out, out_len, info_ptr)
            },
        ))?;
        let table = |layer: i32| -> &[String] {
            let slot = if layer == sys::AICB_LAYER_UI { &self.layers.ui } else { &self.layers.world };
            slot.as_ref().map_or(&[], |f| f.chars.as_slice())
        };
        let image = pixels
            .iter()
            .map(|p| {
                // From<CharacterBuf> for Substr (text.rs:111-119)
                let text = match p.text {
                    sys::AICB_TEXT_EMPTY => ".".to_owned(),
                    sys::AICB_TEXT_INCOMPLETE => "X".to_owned(),
                    sys::AICB_TEXT_ENTERED_SPACE | sys::AICB_TEXT_BLANK => " ".to_owned(),
                    i => table(p.layer).get(i as usize).cloned().unwrap_or_else(|| "#".to_owned()),
                };
                (text, Some(Rgba::new(p.rgba[0], p.rgba[1], p.rgba[2], p.rgba[3])))
            })
            .collect();
        Ok((image, info))
    }

    fn sync_layer(
        backend: &Backend,
        slot: &mut Option<SceneFollower>,
        space: Option<&Handle<Space>>,
        ticket: ReadTicket<'_>,
    ) -> Result<bool, RenderError> {
        // the Option-synchronisation of renderer.rs:124-143
        match (space, &mut *slot) {
            (Some(space), Some(follower)) if *space == follower.space => {}
            (Some(space), slot) => *slot = Some(SceneFollower::new(space.clone())),
            (None, slot) => *slot = None,
        }
        match slot {
            Some(follower) => follower.update(backend, ticket),
            None => Ok(false),
        }
    }
}

impl HeadlessRenderer for B200Renderer {
    fn update(&mut self, read_tickets: Layers<ReadTicket<'_>>, cursor: Option<&Cursor>) -> Result<(), RenderError> {
        self.had_cursor = cursor.is_some(); // the raytracer does not draw the cursor either (renderer.rs:104-105)
        self.cameras.update(read_tickets);
        let world_space = self.cameras.world_space().get();
        Self::sync_layer(&self.backend, &mut self.layers.world, Option::as_ref(&world_space), read_tickets.world)?;
        Self::sync_layer(&self.backend, &mut self.layers.ui, self.cameras.ui_space(), read_tickets.ui)?;
        Ok(())
    }

    fn draw<'a>(&'a mut self, info_text: &'a str) -> BoxFuture<'a, Result<Rendering, RenderError>> {
        Box::pin(async move {
            let cams: &Layers<Camera> = self.cameras.cameras();
            let size = cams.world.viewport().framebuffer_size;
            let mut data = vec![[0u8; 4]; (size.width as usize) * (size.height as usize)];

            // StandardCameras' UiViewState::backdrop (renderer.rs:235-252) and palette::NO_WORLD_TO_SHOW (:474-477)
            let backdrop: Rgba = self.cameras.ui_view_state().backdrop;
            let backdrop_arr: [f32; 4] = backdrop.into();
            let backdrop_ptr: *const [f32; 4] = if backdrop == Rgba::TRANSPARENT { core::ptr::null() } else { &backdrop_arr };
            let no_world: [f32; 4] = palette::NO_WORLD_TO_SHOW.into();

            let mut info = sys::aicb_render_info::default();
            if self.layers.world.is_some() || self.layers.ui.is_some() {
                let (out, out_len) = (data.as_mut_ptr(), data.len());
                let info_ptr: *mut sys::aicb_render_info = &mut info;
                // on a group: aicb_group_render_layers_srgb8, the same pixels from every device
                check(self.with_layers(
                    cams,
                    |world, ui| unsafe {
                        sys::aicb_render_layers_srgb8(world, ui, backdrop_ptr, &no_world, out, out_len, info_ptr)
                    },
                    |world, ui| unsafe {
                        sys::aicb_group_render_layers_srgb8(world, ui, backdrop_ptr, &no_world, out, out_len, info_ptr)
                    },
                ))
                .map_err(to_render_error)?;
            } else {
                // no Space at all: every accumulator is painted NO_WORLD_TO_SHOW (renderer.rs:474-477)
                let px = cams.world.post_process_color(palette::NO_WORLD_TO_SHOW).to_srgb8();
                data.fill(px);
            }

            // draw_info_text (renderer.rs:659-683): outline black, foreground white, over the encoded pixels
            if !info_text.is_empty() {
                all_is_cubes_render::raytracer::draw_info_text(
                    &mut data,
                    cams.world.viewport(),
                    &[[0, 0, 0, 255], [255, 255, 255, 255]],
                    info_text,
                );
            }

            let mut flaws = Flaws::empty(); // as draw_rgba (renderer.rs:293-300)
            if cams.world.options().bloom_intensity != ZeroOne::ZERO {
                flaws |= Flaws::NO_BLOOM;
            }
            if self.had_cursor {
                flaws |= Flaws::NO_CURSOR;
            }
            Ok(Rendering { size, data, flaws, info: Arc::new(B200Info(info)) })
        })
    }
}

/// `ImageInfo` (renderer.rs:609-646) as the library reports it.
#[derive(Clone, Copy, Debug)]
pub struct B200Info(pub sys::aicb_render_info);
impl core::fmt::Display for B200Info {
    fn fmt(&self, f: &mut core::fmt::Formatter<'_>) -> core::fmt::Result {
        write!(f, "Traced {} cubes, {} rays in {:.3} ms on the GPU", self.0.cubes_traced, self.0.rays, self.0.kernel_ms)
    }
}

/// `RendererFactory` for the reference's renderer-agnostic suite (test-renderers/types/src/render.rs:61-82).
#[derive(Clone, Debug)]
pub struct B200Factory {
    ctx: Arc<B200Context>,
}
impl B200Factory {
    pub fn new() -> Result<Self, B200Error> {
        Ok(Self { ctx: B200Context::new(-1)? })
    }
    pub fn renderer_from_cameras(&self, cameras: StandardCameras) -> Box<dyn HeadlessRenderer + Send> {
        Box::new(B200Renderer::new(self.ctx.clone(), cameras))
    }
    pub fn info(&self) -> String {
        format!("libaicb200 ABI {}", unsafe { sys::aicb_abi_version() })
    }
}

/// Snapshot of a `Mutex`-free listener slot, only to keep `Mutex` imported for downstream feature flags.
#[doc(hidden)]
pub type _Unused = Mutex<()>;
