//! `B200Renderer`: the reference's `HeadlessRenderer` (all-is-cubes-render/src/headless.rs:17-44) on top of
//! `libaicb200` — a drop-in for `RtRenderer<()>` (raytracer/renderer.rs:38-355) wherever a
//! `Box<dyn HeadlessRenderer + Send>` is built (test-renderers/types/src/render.rs:61-82,
//! all-is-cubes-desktop/src/record.rs:210-236).
//!
//! * `update()` = `RtRenderer::update` (renderer.rs:96-161): camera sync, then per layer either a full snapshot
//!   (`SpaceRaytracer::new`, sr.rs:64-88 → `aicb_scene_create`) or the `SpaceChange` deltas an
//!   `UpdatingSpaceRaytracer` would apply (updating.rs:107-172 → `aicb_scene_update_blocks` / `_update_cubes`).
//! * `draw()` = `RtRenderer::draw_rgba` (renderer.rs:282-308) with `trace_ray_through_layers` (renderer.rs:454-478)
//!   → `aicb_render_layers_srgb8`; the info text is drawn here over the returned pixels like renderer.rs:659-683.
//!
//! Not compiled in the repository this file ships in (no Rust toolchain there); see ../README.md.

mod convert;

use std::sync::{Arc, Mutex};

use all_is_cubes::character::Cursor;
use all_is_cubes::content::palette;
use all_is_cubes::listen::{self, Listen as _};
use all_is_cubes::math::{Cube, Rgba, ZeroOne};
use all_is_cubes::space::{self, Space, SpaceChange};
use all_is_cubes::universe::{Handle, ReadTicket};
use all_is_cubes::util::maybe_sync::BoxFuture;
use all_is_cubes_b200_sys as sys;
use all_is_cubes_render::camera::{Camera, Layers, StandardCameras};
use all_is_cubes_render::{Flaws, HeadlessRenderer, RenderError, Rendering};

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
    scene: *mut sys::aicb_scene,
    todo: listen::StoreLock<Todo>,
}
// SAFETY: see B200Context.
unsafe impl Send for SceneFollower {}

impl SceneFollower {
    fn new(space: Handle<Space>) -> Self {
        Self {
            space,
            scene: core::ptr::null_mut(),
            todo: listen::StoreLock::new(Todo { listener: true, everything: true, ..Todo::default() }),
        }
    }

    fn update(&mut self, ctx: &B200Context, read_ticket: ReadTicket<'_>) -> Result<bool, RenderError> {
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
        if self.scene.is_null() || todo.everything {
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
            let mut fresh = core::ptr::null_mut();
            check(unsafe { sys::aicb_scene_create(ctx.0, &desc, &mut fresh) }).map_err(to_render_error)?;
            if !self.scene.is_null() {
                unsafe { sys::aicb_scene_destroy(self.scene) };
            }
            self.scene = fresh;
        } else {
            // SpaceChange::BlockIndex / BlockEvaluation: re-run TracingBlock::from_block for those indices (updating.rs:128-150)
            if !todo.blocks.is_empty() {
                let idx: Vec<u16> = todo.blocks.iter().copied().collect();
                let owned: Vec<OwnedBlockDesc> =
                    idx.iter().map(|&i| block_desc_of(&space.block_data()[usize::from(i)])).collect();
                let descs: Vec<sys::aicb_block_desc> = owned.iter().map(OwnedBlockDesc::as_ffi).collect();
                check(unsafe { sys::aicb_scene_update_blocks(self.scene, idx.as_ptr(), descs.as_ptr(), idx.len()) })
                    .map_err(to_render_error)?;
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
                check(unsafe {
                    sys::aicb_scene_update_cubes(self.scene, cubes.as_ptr(), ids.as_ptr(), light.as_ptr(), cubes.len())
                })
                .map_err(to_render_error)?;
            }
        }
        Ok(true)
    }
}
impl Drop for SceneFollower {
    fn drop(&mut self) {
        if !self.scene.is_null() {
            unsafe { sys::aicb_scene_destroy(self.scene) };
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
    ctx: Arc<B200Context>,
    cameras: StandardCameras,
    layers: Layers<Option<SceneFollower>>,
    had_cursor: bool,
}

impl B200Renderer {
    /// == `RtRenderer::new(cameras, size_policy = identity, custom_options = ())` (renderer.rs:65-81)
    pub fn new(ctx: Arc<B200Context>, cameras: StandardCameras) -> Self {
        Self { ctx, cameras, layers: Layers { world: None, ui: None }, had_cursor: false }
    }

    fn sync_layer(
        ctx: &B200Context,
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
            Some(follower) => follower.update(ctx, ticket),
            None => Ok(false),
        }
    }
}

impl HeadlessRenderer for B200Renderer {
    fn update(&mut self, read_tickets: Layers<ReadTicket<'_>>, cursor: Option<&Cursor>) -> Result<(), RenderError> {
        self.had_cursor = cursor.is_some(); // the raytracer does not draw the cursor either (renderer.rs:104-105)
        self.cameras.update(read_tickets);
        let world_space = self.cameras.world_space().get();
        Self::sync_layer(&self.ctx, &mut self.layers.world, Option::as_ref(&world_space), read_tickets.world)?;
        Self::sync_layer(&self.ctx, &mut self.layers.ui, self.cameras.ui_space(), read_tickets.ui)?;
        Ok(())
    }

    fn draw<'a>(&'a mut self, info_text: &'a str) -> BoxFuture<'a, Result<Rendering, RenderError>> {
        Box::pin(async move {
            let cams: &Layers<Camera> = self.cameras.cameras();
            let size = cams.world.viewport().framebuffer_size;
            let mut data = vec![[0u8; 4]; (size.width as usize) * (size.height as usize)];

            let world_cam = camera_of(&cams.world);
            let world_opt = options_of(cams.world.options());
            let ui_cam = camera_of(&cams.ui);
            let ui_opt = options_of(cams.ui.options());
            let world = self.layers.world.as_ref().map(|f| sys::aicb_layer { scene: f.scene, camera: &world_cam, options: &world_opt });
            let ui = self.layers.ui.as_ref().map(|f| sys::aicb_layer { scene: f.scene, camera: &ui_cam, options: &ui_opt });

            // StandardCameras' UiViewState::backdrop (renderer.rs:235-252) and palette::NO_WORLD_TO_SHOW (:474-477)
            let backdrop: Rgba = self.cameras.ui_view_state().backdrop;
            let backdrop_arr: [f32; 4] = backdrop.into();
            let no_world: [f32; 4] = palette::NO_WORLD_TO_SHOW.into();

            let mut info = sys::aicb_render_info::default();
            if world.is_some() || ui.is_some() {
                check(unsafe {
                    sys::aicb_render_layers_srgb8(
                        world.as_ref().map_or(core::ptr::null(), |l| l),
                        ui.as_ref().map_or(core::ptr::null(), |l| l),
                        if backdrop == Rgba::TRANSPARENT { core::ptr::null() } else { &backdrop_arr },
                        &no_world,
                        data.as_mut_ptr(),
                        data.len(),
                        &mut info,
                    )
                })
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
