//! Reference types -> the plain structs of `include/aicb200.h`.

use all_is_cubes::block::{EvaluatedBlock, Evoxels, AIR_EVALUATED};
use all_is_cubes::math::{Face6, GridAab, Rgb, Rgba};
use all_is_cubes::space::{self, LightPhysics, Sky};
use all_is_cubes_b200_sys as sys;
use all_is_cubes_render::camera::{
    AntialiasingOption, Camera, FogOption, GraphicsOptions, LightingOption, ToneMappingOperator, TransparencyOption,
};

pub(crate) fn aab_of(b: GridAab) -> sys::aicb_aab {
    let lo = b.lower_bounds();
    let size = b.size();
    sys::aicb_aab { lower: [lo.x, lo.y, lo.z], size: [size.width, size.height, size.depth] }
}

/// `Sky` (space/sky.rs:16-21); octant order = `(x>=0)<<2 | (y>=0)<<1 | (z>=0)` (sky.rs:36-39).
pub fn sky_of(sky: &Sky) -> sys::aicb_sky {
    let rgb = |c: Rgb| -> [f32; 3] { c.into() };
    match *sky {
        Sky::Uniform(c) => sys::aicb_sky { kind: 0, colors: [rgb(c); 8] },
        Sky::Octants(colors) => sys::aicb_sky { kind: 1, colors: colors.map(rgb) },
        // any future variant: its mean colour, like BlockSky::mean would give the light path
        ref other => sys::aicb_sky { kind: 0, colors: [rgb(other.mean()); 8] },
    }
}

pub(crate) fn light_max_distance_of(light: &LightPhysics) -> u8 {
    match *light {
        LightPhysics::None => 0,
        LightPhysics::Rays { maximum_distance } => maximum_distance,
        _ => 30,
    }
}

/// `aicb_block_desc` with the arrays it points to.
pub struct OwnedBlockDesc {
    indices: Vec<u16>,
    palette: Vec<sys::aicb_voxel>,
    desc: sys::aicb_block_desc,
}
impl OwnedBlockDesc {
    pub fn as_ffi(&self) -> sys::aicb_block_desc {
        let mut d = self.desc;
        d.indices = if self.indices.is_empty() { core::ptr::null() } else { self.indices.as_ptr() };
        d.n_indices = self.indices.len();
        d.palette = self.palette.as_ptr();
        d.n_palette = self.palette.len();
        d
    }
}

/// `TracingBlock::from_block` (sr.rs:579-587) + the `EvaluatedBlock` members light propagation reads
/// (block/eval/evaluated.rs:189-267).
pub fn block_desc_of(data: &space::SpaceBlockData) -> OwnedBlockDesc {
    let ev: &EvaluatedBlock = data.evaluated();
    let voxel = |v: &all_is_cubes::block::Evoxel| {
        let c: [f32; 4] = v.color.into();
        let e: [f32; 3] = v.emission.into();
        let mut flags = if v.selectable { 0 } else { sys::AICB_VOXEL_NOT_SELECTABLE };
        if v.collision == all_is_cubes::block::BlockCollision::None {
            flags |= sys::AICB_VOXEL_NO_COLLISION;
        }
        sys::aicb_voxel { rgba: c, emission: e, flags }
    };
    let (indices, palette, bounds, resolution) = match ev.voxels() {
        // Evoxels::One: indices == NULL (include/aicb200.h, aicb_block_desc)
        voxels if voxels.single_voxel().is_some() => {
            (Vec::new(), vec![voxel(&voxels.single_voxel().unwrap())], GridAab::ORIGIN_CUBE, 1u8)
        }
        voxels => {
            // paletted storage: one u16 per voxel of voxel_bounds, already Z-major (vol.rs:1013-1018)
            let vol = voxels.as_vol_ref();
            let mut palette: Vec<sys::aicb_voxel> = Vec::new();
            let mut lookup = std::collections::HashMap::new();
            let indices = vol
                .as_linear()
                .iter()
                .map(|v| {
                    *lookup.entry((v.color.to_bits(), v.emission.to_bits(), v.selectable, v.collision == all_is_cubes::block::BlockCollision::None)).or_insert_with(|| {
                        palette.push(voxel(v));
                        (palette.len() - 1) as u16
                    })
                })
                .collect();
            (indices, palette, vol.bounds(), u8::from(voxels.resolution()))
        }
    };
    let opaque = ev.opaque();
    let mut opaque_bits = 0u8;
    let mut face_colors = [[0f32; 4]; 6];
    for (i, face) in Face6::ALL.into_iter().enumerate() {
        if opaque[face] {
            opaque_bits |= 1 << i;
        }
        face_colors[i] = ev.face7_color(face.into()).into();
    }
    let color: Rgba = ev.color();
    OwnedBlockDesc {
        indices,
        palette,
        desc: sys::aicb_block_desc {
            resolution,
            is_air: u8::from(*ev == AIR_EVALUATED), // TracingCubeData::always_invisible (sr.rs:547)
            light_opaque_faces: opaque_bits,
            light_visible: u8::from(ev.visible_or_animated()),
            voxel_bounds: aab_of(bounds),
            indices: core::ptr::null(),
            n_indices: 0,
            palette: core::ptr::null(),
            n_palette: 0,
            light_face_colors: face_colors,
            light_color: color.into(),
            light_emission: ev.light_emission().into(),
            flags: if ev.attributes().selectable { 0 } else { sys::AICB_BLOCK_NOT_SELECTABLE },
        },
    }
}

/// What `Camera::project_ndc_into_world` / `post_process_color` need (camera_struct.rs:238-257, 376-382).
/// A `Body` as `aicb_step_bodies` takes it (physics/body.rs: every field through the public accessors;
/// `collision_box_abs()` is `occupying`).
pub fn body_of(body: &all_is_cubes::physics::Body) -> sys::aicb_body {
    let aab = |a: all_is_cubes::math::Aab| {
        let (l, u) = (a.lower_bounds_p(), a.upper_bounds_p());
        [l.x, l.y, l.z, u.x, u.y, u.z]
    };
    let p = body.position();
    let v = body.velocity();
    sys::aicb_body {
        position: [p.x, p.y, p.z],
        velocity: [v.x, v.y, v.z],
        collision_box: aab(body.collision_box_rel()),
        occupying: aab(body.collision_box_abs()),
        flying: u8::from(body.flying),
        noclip: u8::from(body.noclip),
        _pad: [0; 6],
    }
}

/// A stepped `aicb_body` back into `body`: its position and velocity.  `Body::set_position` resets `occupying` to the
/// uncrushed box, which is what the next step's `uncrush` would restore where there is room; the crushed box itself
/// cannot be written from outside the reference's physics module.
pub fn apply_stepped_body(body: &mut all_is_cubes::physics::Body, stepped: &sys::aicb_body) {
    let [x, y, z] = stepped.position;
    body.set_position(all_is_cubes::math::FreePoint::new(x, y, z));
    let [vx, vy, vz] = stepped.velocity;
    body.set_velocity(euclid::vec3(vx, vy, vz));
}

/// An eye's `ViewTransform` (its eye-to-world transform) as `aicb_step_exposure` takes it: `to_transform()` as m11..m44,
/// row-major (euclid `Transform3D::to_array`), what `aicb_view_transform_matrix` computes from its rotation and
/// translation.
pub fn view_transform_of(vt: &all_is_cubes::camera::ViewTransform) -> [f64; 16] {
    vt.to_transform().to_array()
}

pub fn camera_of(camera: &Camera) -> sys::aicb_camera {
    let size = camera.viewport().framebuffer_size;
    sys::aicb_camera {
        inverse_projection_view: camera.inverse_projection_view().to_array(), // euclid Transform3D: m11..m44, row-major
        fb_width: size.width,
        fb_height: size.height,
        exposure: camera.exposure().into_inner(),
        _pad: 0,
    }
}

/// The `GraphicsOptions` fields that affect the raytracer's pixels (graphics_options.rs:28-150), already repaired.
pub fn options_of(options: &GraphicsOptions) -> sys::aicb_options {
    sys::aicb_options {
        fog: match options.fog {
            FogOption::None => 0,
            FogOption::Abrupt => 1,
            FogOption::Compromise => 2,
            FogOption::Physical => 3,
            _ => 1,
        },
        lighting_display: match options.lighting_display {
            LightingOption::None => 0,
            LightingOption::Flat => 1,
            LightingOption::Coarse => 2,
            LightingOption::Linear => 3,
            LightingOption::Smoothstep => 4,
            LightingOption::Bounce { .. } => 5,
            _ => 3,
        },
        transparency: match options.transparency {
            TransparencyOption::Surface => 0,
            TransparencyOption::Volumetric => 1,
            TransparencyOption::Threshold(_) => 2,
            _ => 1,
        },
        antialiasing_always: u8::from(matches!(options.antialiasing, AntialiasingOption::Always)),
        tone_mapping: match options.tone_mapping {
            ToneMappingOperator::Clamp => 0,
            ToneMappingOperator::Reinhard => 1,
            _ => 0,
        },
        debug_pixel_cost: u8::from(options.debug_pixel_cost),
        include_sky: 1,
        bounce_samples: match options.lighting_display {
            LightingOption::Bounce { samples } => samples.max(1),
            _ => 0,
        },
        transparency_threshold: match options.transparency {
            TransparencyOption::Threshold(t) => t.into_inner(),
            _ => 0.0,
        },
        maximum_intensity: options.maximum_intensity.into_inner(),
        view_distance: options.view_distance.into_inner(),
    }
}
