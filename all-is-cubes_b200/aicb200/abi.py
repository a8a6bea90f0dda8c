"""ctypes mirror of include/aicb200.h (plain data only; no compute)."""
import ctypes as C

import numpy as np

ABI_VERSION = 28

BLOCKS_DERIVE_LIGHT = 1

OK, ERR_INVALID, ERR_OOM, ERR_CUDA, ERR_UNSUPPORTED, ERR_BUSY, ERR_RETRY = range(7)
STATUS_NAMES = {0: "OK", 1: "ERR_INVALID", 2: "ERR_OOM", 3: "ERR_CUDA", 4: "ERR_UNSUPPORTED", 5: "ERR_BUSY", 6: "ERR_RETRY"}

FACE_WITHIN, FACE_NX, FACE_NY, FACE_NZ, FACE_PX, FACE_PY, FACE_PZ = range(7)
FOG_NONE, FOG_ABRUPT, FOG_COMPROMISE, FOG_PHYSICAL = range(4)
LIGHT_NONE, LIGHT_FLAT, LIGHT_COARSE, LIGHT_LINEAR, LIGHT_SMOOTHSTEP, LIGHT_BOUNCE = range(6)
TRANSPARENCY_SURFACE, TRANSPARENCY_VOLUMETRIC, TRANSPARENCY_THRESHOLD = range(3)
TONE_CLAMP, TONE_REINHARD = range(2)


class Aab(C.Structure):
    _fields_ = [("lower", C.c_int32 * 3), ("size", C.c_uint32 * 3)]


class Voxel(C.Structure):
    _fields_ = [("rgba", C.c_float * 4), ("emission", C.c_float * 3), ("flags", C.c_uint32)]


class BlockDesc(C.Structure):
    _fields_ = [
        ("resolution", C.c_uint8),
        ("is_air", C.c_uint8),
        ("light_opaque_faces", C.c_uint8),
        ("light_visible", C.c_uint8),
        ("voxel_bounds", Aab),
        ("indices", C.c_void_p),
        ("n_indices", C.c_size_t),
        ("palette", C.c_void_p),
        ("n_palette", C.c_size_t),
        ("light_face_colors", (C.c_float * 4) * 6),
        ("light_color", C.c_float * 4),
        ("light_emission", C.c_float * 3),
        ("flags", C.c_uint32),
    ]


class BlockLight(C.Structure):
    """aicb_block_light: compute_derived's light fields of one block, as aicb_block_desc's light_* members take them."""
    _fields_ = [
        ("face_colors", (C.c_float * 4) * 6),
        ("color", C.c_float * 4),
        ("emission", C.c_float * 3),
        ("opaque_faces", C.c_uint8),
        ("visible", C.c_uint8),
        ("_pad", C.c_uint8 * 2),
    ]


class Sky(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("colors", (C.c_float * 3) * 8)]


class SceneDesc(C.Structure):
    _fields_ = [
        ("bounds", Aab),
        ("block_ids", C.c_void_p),
        ("light", C.c_void_p),
        ("blocks", C.POINTER(BlockDesc)),
        ("n_blocks", C.c_size_t),
        ("sky", Sky),
        ("light_max_distance", C.c_uint8),
        ("_pad", C.c_uint8 * 7),
    ]


class CameraData(C.Structure):
    _fields_ = [
        ("inverse_projection_view", C.c_double * 16),
        ("fb_width", C.c_uint32),
        ("fb_height", C.c_uint32),
        ("exposure", C.c_float),
        ("_pad", C.c_uint32),
    ]


# aicb_camera as a numpy structured dtype: the camera table of a batch of views (draw_views with device=True)
CAMERA_DTYPE = np.dtype([("inverse_projection_view", "<f8", (16,)), ("fb_width", "<u4"), ("fb_height", "<u4"),
                         ("exposure", "<f4"), ("_pad", "<u4")])
assert CAMERA_DTYPE.itemsize == C.sizeof(CameraData) == 144


class Options(C.Structure):
    _fields_ = [
        ("fog", C.c_uint8),
        ("lighting_display", C.c_uint8),
        ("transparency", C.c_uint8),
        ("antialiasing_always", C.c_uint8),
        ("tone_mapping", C.c_uint8),
        ("debug_pixel_cost", C.c_uint8),
        ("include_sky", C.c_uint8),
        ("bounce_samples", C.c_uint8),
        ("transparency_threshold", C.c_float),
        ("maximum_intensity", C.c_float),
        ("view_distance", C.c_double),
    ]


class Shard(C.Structure):
    _fields_ = [("strip_rows", C.c_uint32), ("index", C.c_uint32), ("count", C.c_uint32)]


class RenderInfo(C.Structure):
    _fields_ = [
        ("cubes_traced", C.c_uint64),
        ("rays", C.c_uint64),
        ("algorithmic_bytes", C.c_uint64),
        ("counters", C.c_uint64 * 6),
        ("kernel_ms", C.c_float),
        ("flaws", C.c_uint16),
        ("ray_order", C.c_uint16),
        ("stage_ms", C.c_float * 4),
    ]


class Hit(C.Structure):
    _fields_ = [("cube", C.c_int32 * 3), ("voxel", C.c_int32 * 3), ("resolution", C.c_int32), ("face", C.c_int32)]


class LightRay(C.Structure):
    _fields_ = [("trigger_cube", C.c_int32 * 3), ("value_cube", C.c_int32 * 3), ("value", C.c_uint8 * 4),
                ("light_from_struck_face", C.c_float * 3), ("_pad", C.c_uint32)]


class LightUpdatesInfo(C.Structure):
    """aicb_light_updates_info: LightUpdatesInfo (space/light/updater.rs:970-984) of one light step."""
    _fields_ = [("update_count", C.c_uint64), ("queue_count", C.c_uint64), ("max_update_difference", C.c_uint8),
                ("max_queue_priority", C.c_uint8), ("_pad", C.c_uint8 * 6)]


# Every symbol include/aicb200.h declares (tests check the built library exports all of them).
class Layer(C.Structure):
    _fields_ = [("scene", C.c_void_p), ("camera", C.POINTER(CameraData)), ("options", C.POINTER(Options))]


class GroupLayer(C.Structure):
    _fields_ = [("scene", C.c_void_p), ("camera", C.POINTER(CameraData)), ("options", C.POINTER(Options))]


TEXT_ENTERED_SPACE, TEXT_EMPTY, TEXT_INCOMPLETE, TEXT_BLANK = -1, -2, -3, -4
LAYER_NONE, LAYER_WORLD, LAYER_UI = 0, 1, 2


class TerminalPixel(C.Structure):
    _fields_ = [("rgba", C.c_float * 4), ("text", C.c_int32), ("layer", C.c_int32)]


class DeviceOutputs(C.Structure):
    """aicb_device_outputs: nullable device pointers of the device-output calls, their length and full_frame."""
    _fields_ = [("srgb8", C.c_void_p), ("rgba16f", C.c_void_p), ("colorbuf", C.c_void_p), ("depth", C.c_void_p),
                ("hit", C.c_void_p), ("steps", C.c_void_p), ("text", C.c_void_p), ("texel_rgba16f", C.c_void_p),
                ("texel_depth", C.c_void_p), ("terminal", C.c_void_p), ("len", C.c_size_t), ("full_frame", C.c_uint32),
                ("_pad", C.c_uint32)]


TEXTURE_INCREMENTAL, TEXTURE_CONSISTENT = 1, 2


class TextureTargetInfo(C.Structure):
    """aicb_texture_target_info: a texture target's size, strategy, dirty_pixels, pick position and cycle_length."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("strategy", C.c_uint32), ("_pad", C.c_uint32),
                ("dirty_pixels", C.c_uint64), ("next_pick", C.c_uint64), ("cycle_length", C.c_uint64)]


VOXEL_NOT_SELECTABLE = 1   # aicb_voxel::flags
VOXEL_NO_COLLISION = 2     # aicb_voxel::flags
BLOCK_NOT_SELECTABLE = 1   # aicb_block_desc::flags
CURSOR_NONE = 0xFFFFFFFF
CURSOR_OUTSIDE = 0xFFFFFFFE


class Cursor(C.Structure):
    """aicb_cursor: Cursor + its CubeSnapshots (cursor.rs:111-149), 80 bytes."""
    _fields_ = [("point_entered", C.c_double * 3), ("distance", C.c_double), ("cube", C.c_int32 * 3),
                ("preceding_cube", C.c_int32 * 3), ("block_id", C.c_uint32), ("preceding_block_id", C.c_uint32),
                ("light", C.c_uint8 * 4), ("preceding_light", C.c_uint8 * 4), ("face_entered", C.c_uint8),
                ("face_selected", C.c_uint8), ("layer", C.c_uint8), ("_pad", C.c_uint8 * 5)]


# aicb_cursor as a numpy structured dtype (the arrays the cursor calls return)
CURSOR_DTYPE = np.dtype([("point_entered", "<f8", (3,)), ("distance", "<f8"), ("cube", "<i4", (3,)),
                         ("preceding_cube", "<i4", (3,)), ("block_id", "<u4"), ("preceding_block_id", "<u4"),
                         ("light", "u1", (4,)), ("preceding_light", "u1", (4,)), ("face_entered", "u1"),
                         ("face_selected", "u1"), ("layer", "u1"), ("_pad", "u1", (5,))])
assert CURSOR_DTYPE.itemsize == 80


CONTACT_NONE, CONTACT_BLOCK, CONTACT_VOXEL = 0, 1, 2
UNCRUSH_NOT_NEEDED, UNCRUSH_NOT_POSSIBLE, UNCRUSH_COMPLETE, UNCRUSH_PARTIAL = 0, 1, 2, 3
AXIS_NONE = 0xFF
BODY_INVALID = 1
BODY_CONTACTS_TRUNCATED = 2
BODY_NO_PENETRATION = 4
BODY_SLIDING_UNFINISHED = 8
BODY_CRUSH_UNFINISHED = 16

# aicb_body, aicb_contact and aicb_body_step_info as numpy structured dtypes (what step_bodies takes and returns)
BODY_DTYPE = np.dtype([("position", "<f8", (3,)), ("velocity", "<f8", (3,)), ("collision_box", "<f8", (6,)),
                       ("occupying", "<f8", (6,)), ("flying", "u1"), ("noclip", "u1"), ("_pad", "u1", (6,))])
assert BODY_DTYPE.itemsize == 152
CONTACT_DTYPE = np.dtype([("cube", "<i4", (3,)), ("voxel", "<i4", (3,)), ("kind", "u1"), ("face", "u1"),
                          ("resolution", "u1"), ("_pad", "u1")])
assert CONTACT_DTYPE.itemsize == 28
MOVE_SEGMENT_DTYPE = np.dtype([("delta_position", "<f8", (3,)), ("stopped_by", CONTACT_DTYPE), ("_pad", "<u4")])
assert MOVE_SEGMENT_DTYPE.itemsize == 56
BODY_STEP_INFO_DTYPE = np.dtype([("move_segments", MOVE_SEGMENT_DTYPE, (3,)), ("push_out", "<f8", (3,)),
                                 ("initial_crush", "<f8", (6,)), ("delta_v", "<f8", (3,)),
                                 ("already_colliding", CONTACT_DTYPE), ("n_contacts", "<u4"), ("status", "<u4"),
                                 ("quiescent", "u1"), ("has_push_out", "u1"), ("uncrush", "u1"),
                                 ("uncrush_axes", "u1", (3,)), ("_pad", "u1", (6,))])
assert BODY_STEP_INFO_DTYPE.itemsize == 312

# aicb_exposure_state as a numpy structured dtype (what step_exposure takes and returns)
EXPOSURE_STATE_DTYPE = np.dtype([("luminance_samples", "<f4", (100,)), ("luminance_sample_index", "<u4"),
                                 ("exposure_log", "<f4")])
assert EXPOSURE_STATE_DTYPE.itemsize == 408

# aicb_eye as a numpy structured dtype (what step_eyes and eye_views take): CharacterEye + PreviousBodyVelocity
EYE_DTYPE = np.dtype([("displacement_pos", "<f8", (3,)), ("displacement_vel", "<f8", (3,)),
                      ("previous_body_velocity", "<f8", (3,))])
assert EYE_DTYPE.itemsize == 72


class EyeViewParams(C.Structure):
    """aicb_eye_view_params: what the world camera of a batch of eyes takes from GraphicsOptions and the Viewport."""
    _fields_ = [("fov_y_degrees", C.c_double), ("view_distance", C.c_double), ("nominal_width", C.c_double),
                ("nominal_height", C.c_double), ("fb_width", C.c_uint32), ("fb_height", C.c_uint32),
                ("fixed_exposure", C.c_float), ("automatic_exposure", C.c_uint8), ("lighting_display", C.c_uint8),
                ("_pad", C.c_uint8 * 2)]


EYE_VIEW_PARAMS = EyeViewParams
assert C.sizeof(EYE_VIEW_PARAMS) == 48
EYE_NOT_INVERTIBLE = 1   # aicb_eye_views_device status


EXPORTED_SYMBOLS = [
    "aicb_abi_version",
    "aicb_ctx_create",
    "aicb_ctx_destroy",
    "aicb_ctx_stage_timing",
    "aicb_ctx_device",
    "aicb_last_error",
    "aicb_derive_block_light",
    "aicb_scene_create",
    "aicb_scene_update_cubes",
    "aicb_scene_update_region",
    "aicb_scene_update_blocks",
    "aicb_scene_append_blocks",
    "aicb_scene_fill_uniform",
    "aicb_scene_upload_light",
    "aicb_scene_destroy",
    "aicb_scene_device_bytes",
    "aicb_scene_set_physics",
    "aicb_scene_update_cubes_device",
    "aicb_scene_update_region_device",
    "aicb_scene_upload_light_device",
    "aicb_scene_download_ids_device",
    "aicb_light_edit_cubes_device",
    "aicb_light_edit_region_device",
    "aicb_light_download_device",
    "aicb_scene_update_blocks_device",
    "aicb_scene_append_blocks_device",
    "aicb_scene_create_device",
    "aicb_scene_fill_uniform_device",
    "aicb_shard_pixel_count",
    "aicb_render_srgb8",
    "aicb_render_rgba16f",
    "aicb_render_colorbuf",
    "aicb_render_text",
    "aicb_render_layers_srgb8",
    "aicb_render_layers_texture",
    "aicb_render_layers_terminal",
    "aicb_ortho_image_size",
    "aicb_render_orthographic",
    "aicb_render_srgb8_device",
    "aicb_render_srgb8_device_frame",
    "aicb_render_finish",
    "aicb_render_device",
    "aicb_trace_rays_device",
    "aicb_render_layers_device",
    "aicb_render_views_srgb8",
    "aicb_render_views_rgba16f",
    "aicb_render_views_colorbuf",
    "aicb_render_views_text",
    "aicb_render_views_device",
    "aicb_frame_create",
    "aicb_frame_open",
    "aicb_frame_close",
    "aicb_frame_read",
    "aicb_frame_signal",
    "aicb_frame_wait_arrived",
    "aicb_frame_release",
    "aicb_frame_wait_consumed",
    "aicb_frame_timed_out",
    "aicb_trace_rays",
    "aicb_camera_look_at",
    "aicb_camera_from_view",
    "aicb_eye_for_look_at",
    "aicb_camera_project_ndc",
    "aicb_view_transform_matrix",
    "aicb_cursor_raycast",
    "aicb_cursor_raycast_device",
    "aicb_project_cursor",
    "aicb_group_cursor_raycast",
    "aicb_group_cursor_raycast_device",
    "aicb_group_project_cursor",
    "aicb_step_bodies",
    "aicb_step_bodies_device",
    "aicb_group_step_bodies",
    "aicb_group_step_bodies_device",
    "aicb_step_exposure",
    "aicb_step_exposure_device",
    "aicb_group_step_exposure",
    "aicb_group_step_exposure_device",
    "aicb_look_rotation",
    "aicb_step_eyes_device",
    "aicb_eye_views_device",
    "aicb_group_step_eyes_device",
    "aicb_group_eye_views_device",
    "aicb_light_chart",
    "aicb_light_chart_chains",
    "aicb_light_fast_evaluate",
    "aicb_light_compute",
    "aicb_light_compute_debug",
    "aicb_light_evaluate",
    "aicb_light_update_from_queue",
    "aicb_light_edit_cubes",
    "aicb_light_edit_and_propagate",
    "aicb_light_edit_region",
    "aicb_light_relight_blocks",
    "aicb_light_download",
    "aicb_light_queue_uninitialized",
    "aicb_light_queue_region",
    "aicb_light_download_queue",
    "aicb_light_stats",
    "aicb_light_changes_count",
    "aicb_light_take_changes",
    "aicb_group_create",
    "aicb_group_destroy",
    "aicb_group_size",
    "aicb_group_scene_create",
    "aicb_group_scene_destroy",
    "aicb_group_scene_update_cubes",
    "aicb_group_scene_update_region",
    "aicb_group_render_srgb8",
    "aicb_group_scene_update_blocks",
    "aicb_group_scene_upload_light",
    "aicb_group_scene_set_physics",
    "aicb_group_scene_append_blocks",
    "aicb_group_scene_fill_uniform",
    "aicb_group_scene_update_cubes_device",
    "aicb_group_scene_update_region_device",
    "aicb_group_scene_upload_light_device",
    "aicb_group_scene_download_ids_device",
    "aicb_group_light_edit_cubes_device",
    "aicb_group_light_edit_region_device",
    "aicb_group_light_download_device",
    "aicb_group_scene_update_blocks_device",
    "aicb_group_scene_append_blocks_device",
    "aicb_group_scene_create_device",
    "aicb_group_scene_fill_uniform_device",
    "aicb_group_render_layers_srgb8",
    "aicb_group_render_layers_texture",
    "aicb_group_render_layers_terminal",
    "aicb_group_render_colorbuf",
    "aicb_group_render_rgba16f",
    "aicb_group_trace_rays",
    "aicb_group_render_text",
    "aicb_group_ortho_image_size",
    "aicb_group_render_orthographic",
    "aicb_group_render_device",
    "aicb_group_trace_rays_device",
    "aicb_group_render_layers_device",
    "aicb_group_render_views_srgb8",
    "aicb_group_render_views_rgba16f",
    "aicb_group_render_views_colorbuf",
    "aicb_group_render_views_text",
    "aicb_group_render_views_device",
    "aicb_texture_target_create",
    "aicb_texture_target_destroy",
    "aicb_texture_target_resize",
    "aicb_texture_target_mark_dirty",
    "aicb_texture_target_trace",
    "aicb_texture_target_state",
    "aicb_texture_target_picks",
    "aicb_texture_target_buffers",
    "aicb_texture_target_read",
    "aicb_group_texture_target_create",
    "aicb_group_texture_target_destroy",
    "aicb_group_texture_target_resize",
    "aicb_group_texture_target_mark_dirty",
    "aicb_group_texture_target_trace",
    "aicb_group_texture_target_state",
    "aicb_group_texture_target_picks",
    "aicb_group_texture_target_buffers",
    "aicb_group_texture_target_read",
    "aicb_group_light_fast_evaluate",
    "aicb_group_light_compute",
    "aicb_group_light_compute_debug",
    "aicb_group_light_evaluate",
    "aicb_group_light_update_from_queue",
    "aicb_group_light_edit_and_propagate",
    "aicb_group_light_edit_cubes",
    "aicb_group_light_edit_region",
    "aicb_group_light_relight_blocks",
    "aicb_group_light_download",
    "aicb_group_light_queue_uninitialized",
    "aicb_group_light_queue_region",
    "aicb_group_light_download_queue",
    "aicb_group_light_stats",
    "aicb_group_light_changes_count",
    "aicb_group_light_take_changes",
]
