"""aicb200 — Python binding over the C ABI of libaicb200.so.

Mirrors the reference's raytracer surface (names and argument meaning):
`GraphicsOptions` (all-is-cubes-render/src/camera/graphics_options.rs:28), `Viewport`
(camera/viewport.rs:24), `Camera` (camera/camera_struct.rs:43), `SpaceRaytracer`
(raytracer/sr.rs:51), `RtRenderer` / `HeadlessRenderer` (raytracer/renderer.rs:35,
headless.rs:17), `Rendering` (headless.rs:52).  `Space`/`Block` here are only the flattened
snapshot the raytracer reads (SpaceRaytracer::new, sr.rs:64-88) — not the reference's world model.

This module contains no compute: every pixel comes from the CUDA kernels behind the C ABI.
If the library is missing or there is no GPU the calls fail loudly (no CPU fallback).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
import os
from typing import Optional, Sequence

import numpy as np

from . import abi
from .abi import (FOG_ABRUPT, FOG_COMPROMISE, FOG_NONE, FOG_PHYSICAL, LIGHT_BOUNCE, LIGHT_COARSE, LIGHT_FLAT, LIGHT_LINEAR,
                  LIGHT_NONE, LIGHT_SMOOTHSTEP, TONE_CLAMP, TONE_REINHARD, TRANSPARENCY_SURFACE,
                  TRANSPARENCY_THRESHOLD, TRANSPARENCY_VOLUMETRIC)

PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.environ.get("AICB200_LIB") or os.path.join(PKG_DIR, "libaicb200.so")  # override: kernel experiments only
LIGHT_RAY_DTYPE = np.dtype(abi.LightRay)   # aicb_light_ray: one ray of light_compute_debug


class AicbError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"{abi.STATUS_NAMES.get(status, status)}: {message}")
        self.status = status


_lib = None


def load_library() -> C.CDLL:
    """Load libaicb200.so (built in-tree by __graft_entry__.build()). Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    lib.aicb_abi_version.restype = C.c_uint32
    lib.aicb_last_error.restype = C.c_char_p
    lib.aicb_ctx_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.aicb_ctx_destroy.argtypes = [C.c_void_p]
    lib.aicb_ctx_stage_timing.argtypes = [C.c_void_p, C.c_int]
    lib.aicb_ctx_device.argtypes = [C.c_void_p]
    lib.aicb_scene_create.argtypes = [C.c_void_p, C.POINTER(abi.SceneDesc), C.POINTER(C.c_void_p)]
    lib.aicb_scene_destroy.argtypes = [C.c_void_p]
    lib.aicb_scene_device_bytes.argtypes = [C.c_void_p]
    lib.aicb_scene_device_bytes.restype = C.c_uint64
    lib.aicb_shard_pixel_count.argtypes = [C.POINTER(abi.CameraData), C.POINTER(abi.Shard)]
    lib.aicb_shard_pixel_count.restype = C.c_size_t
    lib.aicb_render_srgb8.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                      C.POINTER(abi.Shard), C.c_void_p, C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_render_colorbuf.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                         C.POINTER(abi.Shard), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_render_rgba16f.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                        C.POINTER(abi.Shard), C.c_void_p, C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_render_srgb8_device.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                             C.POINTER(abi.Shard), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.aicb_render_srgb8_device_frame.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                                   C.POINTER(abi.Shard), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.aicb_frame_create.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.c_void_p]
    lib.aicb_frame_open.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.aicb_frame_close.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.aicb_frame_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.aicb_frame_signal.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.aicb_frame_wait_arrived.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.aicb_frame_release.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.aicb_frame_wait_consumed.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.aicb_frame_timed_out.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32)]
    lib.aicb_render_finish.argtypes = [C.c_void_p, C.POINTER(abi.RenderInfo)]
    lib.aicb_camera_look_at.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_double,
                                        C.c_double, C.c_double, C.c_uint32, C.c_uint32, C.c_float,
                                        C.POINTER(abi.CameraData)]
    lib.aicb_camera_from_view.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_double,
                                          C.c_double, C.c_double, C.c_uint32, C.c_uint32, C.c_float,
                                          C.POINTER(abi.CameraData)]
    lib.aicb_eye_for_look_at.argtypes = [C.POINTER(abi.Aab), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.aicb_eye_for_look_at.restype = None
    lib.aicb_camera_project_ndc.argtypes = [C.POINTER(abi.CameraData), C.c_double, C.c_double,
                                            C.POINTER(C.c_double)]
    lib.aicb_camera_project_ndc.restype = None
    lib.aicb_view_transform_matrix.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.aicb_view_transform_matrix.restype = None
    lib.aicb_light_download.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.aicb_render_layers_srgb8.argtypes = [C.POINTER(abi.Layer), C.POINTER(abi.Layer), C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_render_layers_texture.argtypes = [C.POINTER(abi.Layer), C.POINTER(abi.Layer), C.c_void_p, C.c_void_p,
                                               C.POINTER(C.c_double), C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                               C.POINTER(abi.RenderInfo)]
    lib.aicb_render_layers_terminal.argtypes = [C.POINTER(abi.Layer), C.POINTER(abi.Layer), C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_create.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p)]
    lib.aicb_group_destroy.argtypes = [C.c_void_p]
    lib.aicb_group_destroy.restype = None
    lib.aicb_group_size.argtypes = [C.c_void_p]
    lib.aicb_group_scene_create.argtypes = [C.c_void_p, C.POINTER(abi.SceneDesc), C.POINTER(C.c_void_p)]
    for name in ("aicb_scene_create_device", "aicb_group_scene_create_device"):
        getattr(lib, name).argtypes = [C.c_void_p, C.POINTER(abi.SceneDesc), C.c_uint32, C.c_void_p,
                                       C.POINTER(C.c_void_p)]
    lib.aicb_group_scene_destroy.argtypes = [C.c_void_p]
    lib.aicb_group_scene_destroy.restype = None
    lib.aicb_group_render_srgb8.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                            C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_layers_srgb8.argtypes = [C.POINTER(abi.GroupLayer), C.POINTER(abi.GroupLayer), C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_layers_texture.argtypes = [C.POINTER(abi.GroupLayer), C.POINTER(abi.GroupLayer), C.c_void_p,
                                                     C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_size_t,
                                                     C.c_void_p, C.c_void_p, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_layers_terminal.argtypes = [C.POINTER(abi.GroupLayer), C.POINTER(abi.GroupLayer), C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_colorbuf.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                               C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_rgba16f.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p,
                                              C.c_size_t, C.POINTER(abi.RenderInfo)]
    for prefix in ("aicb_", "aicb_group_"):
        for kind in ("srgb8", "rgba16f", "text"):
            getattr(lib, prefix + "render_views_" + kind).argtypes = [
                C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), C.c_void_p, C.c_size_t,
                C.POINTER(abi.RenderInfo)]
        getattr(lib, prefix + "render_views_colorbuf").argtypes = [
            C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
            C.c_size_t, C.POINTER(abi.RenderInfo)]
    lib.aicb_render_views_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                             C.POINTER(abi.Options), C.POINTER(abi.DeviceOutputs), C.c_void_p]
    lib.aicb_group_render_views_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                                   C.POINTER(abi.Options), C.POINTER(abi.DeviceOutputs), C.c_void_p,
                                                   C.POINTER(abi.RenderInfo)]
    lib.aicb_light_chart.argtypes = [C.c_void_p, C.c_void_p]
    lib.aicb_light_chart.restype = C.c_uint32
    outs = C.POINTER(abi.DeviceOutputs)
    lib.aicb_render_device.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options),
                                       C.POINTER(abi.Shard), outs, C.c_void_p]
    lib.aicb_trace_rays_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), outs,
                                           C.c_void_p]
    lib.aicb_render_layers_device.argtypes = [C.POINTER(abi.Layer), C.POINTER(abi.Layer), C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_size_t, outs, C.c_void_p]
    lib.aicb_group_render_device.argtypes = [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), outs,
                                             C.c_void_p, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_trace_rays_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), outs,
                                                 C.c_void_p, C.POINTER(abi.RenderInfo)]
    lib.aicb_group_render_layers_device.argtypes = [C.POINTER(abi.GroupLayer), C.POINTER(abi.GroupLayer), C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, outs, C.c_void_p,
                                                    C.POINTER(abi.RenderInfo)]
    lib.aicb_group_light_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    lib.aicb_derive_block_light.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    for prefix in ("aicb_", "aicb_group_"):
        getattr(lib, prefix + "cursor_raycast").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        getattr(lib, prefix + "cursor_raycast_device").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                                  C.c_void_p, C.c_void_p]
    for prefix in ("aicb_", "aicb_group_"):
        getattr(lib, prefix + "step_bodies").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double,
                                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        getattr(lib, prefix + "step_bodies_device").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                               C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                                               C.c_uint32, C.c_void_p]
    for prefix in ("aicb_", "aicb_group_"):
        getattr(lib, prefix + "step_exposure").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double,
                                                          C.c_void_p]
        getattr(lib, prefix + "step_exposure_device").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                                 C.c_double, C.c_void_p, C.c_void_p]
    lib.aicb_look_rotation.argtypes = [C.c_double, C.c_double, C.c_void_p]
    lib.aicb_look_rotation.restype = None
    for prefix in ("aicb_", "aicb_group_"):
        getattr(lib, prefix + "step_eyes_device").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                             C.c_double, C.c_void_p]
        getattr(lib, prefix + "eye_views_device").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                             C.c_void_p, C.c_size_t, C.POINTER(abi.EyeViewParams),
                                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                             C.c_void_p]
    lib.aicb_project_cursor.argtypes = [C.POINTER(abi.Layer), C.POINTER(abi.Layer), C.c_void_p, C.c_size_t,
                                        C.c_double, C.c_void_p]
    lib.aicb_group_project_cursor.argtypes = [C.POINTER(abi.GroupLayer), C.POINTER(abi.GroupLayer), C.c_void_p,
                                              C.c_size_t, C.c_double, C.c_void_p]
    # the calls of _Scene: a group scene's form of aicb_<name> is aicb_group_<name>, with the same arguments
    u64, u8, size = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_size_t)
    info = C.POINTER(abi.RenderInfo)
    for name, argtypes in {
        "trace_rays": [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(abi.Options), C.c_void_p, C.c_void_p, C.c_void_p,
                       C.c_void_p, info],
        "render_text": [C.c_void_p, C.POINTER(abi.CameraData), C.POINTER(abi.Options), C.c_void_p, C.c_size_t, info],
        "ortho_image_size": [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)],
        "render_orthographic": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, info],
        "scene_update_cubes": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t],
        "scene_update_region": [C.c_void_p, C.POINTER(abi.Aab), C.c_void_p, C.c_uint16, C.c_void_p],
        "scene_update_blocks": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t],
        "scene_append_blocks": [C.c_void_p, C.c_void_p, C.c_size_t],
        "scene_fill_uniform": [C.c_void_p, C.c_void_p],
        "scene_upload_light": [C.c_void_p, C.c_void_p, C.c_size_t],
        "scene_set_physics": [C.c_void_p, C.POINTER(abi.Sky), C.c_uint8],
        "light_fast_evaluate": [C.c_void_p],
        "light_compute": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
        "light_compute_debug": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                size],
        "light_evaluate": [C.c_void_p, C.c_uint8, u64, u8, u64],
        "light_update_from_queue": [C.c_void_p, C.c_uint64, C.POINTER(abi.LightUpdatesInfo)],
        "light_edit_cubes": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, size],
        "light_edit_and_propagate": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint8, u64, u8],
        "light_edit_region": [C.c_void_p, C.POINTER(abi.Aab), C.c_void_p, C.c_uint16, size],
        "light_relight_blocks": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint8, u64, u8],
        "light_stats": [C.c_void_p, u64],
        "light_queue_uninitialized": [C.c_void_p, size],
        "light_queue_region": [C.c_void_p, C.POINTER(abi.Aab), C.c_uint8],
        "light_download_queue": [C.c_void_p, C.c_void_p, C.c_size_t, size],
        "light_changes_count": [C.c_void_p, size],
        "light_take_changes": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, size],
        "scene_update_cubes_device": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
        "scene_update_region_device": [C.c_void_p, C.POINTER(abi.Aab), C.c_void_p, C.c_uint16, C.c_void_p, C.c_void_p],
        "scene_upload_light_device": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
        "scene_download_ids_device": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
        "light_edit_cubes_device": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, size, C.c_void_p],
        "light_edit_region_device": [C.c_void_p, C.POINTER(abi.Aab), C.c_void_p, C.c_uint16, size, C.c_void_p],
        "light_download_device": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p],
        "scene_update_blocks_device": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p],
        "scene_append_blocks_device": [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p],
        "scene_fill_uniform_device": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p],
    }.items():
        for prefix in ("aicb_", "aicb_group_"):
            getattr(lib, prefix + name).argtypes = argtypes
    # the texture targets: aicb_texture_target_<name> and aicb_group_texture_target_<name>, the layers aside
    for name, argtypes in {
        "create": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_void_p)],
        "destroy": [C.c_void_p],
        "resize": [C.c_void_p, C.c_uint32, C.c_uint32],
        "mark_dirty": [C.c_void_p],
        "state": [C.c_void_p, C.POINTER(abi.TextureTargetInfo)],
        "picks": [C.c_void_p, C.c_uint64, C.c_size_t, C.c_void_p],
        "buffers": [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)],
        "read": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t],
    }.items():
        for prefix in ("aicb_texture_target_", "aicb_group_texture_target_"):
            getattr(lib, prefix + name).argtypes = argtypes
    lib.aicb_texture_target_destroy.restype = None
    lib.aicb_group_texture_target_destroy.restype = None
    for prefix, layer in (("aicb_", abi.Layer), ("aicb_group_", abi.GroupLayer)):
        getattr(lib, prefix + "texture_target_trace").argtypes = [
            C.c_void_p, C.POINTER(layer), C.POINTER(layer), C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_size_t,
            size, info]
    if lib.aicb_abi_version() != abi.ABI_VERSION:
        raise RuntimeError("libaicb200.so ABI version mismatch")
    _lib = lib
    return lib


# The camera matrices (host-only code, all-is-cubes_b200/host/camera.cpp) are reached through the C ABI of
# libaicb200.so by default.  bench.py's reference arm must not load the product library at all, so the same host
# source is also compiled into the oracle library under orc_* names; use_camera_library() points Camera at it.
_camera_lib = None
_camera_prefix = "aicb_"


def use_camera_library(lib, prefix: str):
    """Route Camera / eye_for_look_at through another shared library exporting <prefix>camera_look_at,
    <prefix>camera_from_view, <prefix>eye_for_look_at, <prefix>camera_project_ndc (same signatures)."""
    global _camera_lib, _camera_prefix
    for name in ("camera_look_at", "camera_from_view"):
        fn = getattr(lib, prefix + name)
        fn.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_double, C.c_double, C.c_double,
                       C.c_uint32, C.c_uint32, C.c_float, C.POINTER(abi.CameraData)]
        fn.restype = C.c_int
    fn = getattr(lib, prefix + "eye_for_look_at")
    fn.argtypes = [C.POINTER(abi.Aab), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    fn.restype = None
    fn = getattr(lib, prefix + "camera_project_ndc")
    fn.argtypes = [C.POINTER(abi.CameraData), C.c_double, C.c_double, C.POINTER(C.c_double)]
    fn.restype = None
    _camera_lib, _camera_prefix = lib, prefix


def _cam(name: str):
    lib = _camera_lib if _camera_lib is not None else load_library()
    return getattr(lib, _camera_prefix + name)


def _check_cam(status: int):
    if status != abi.OK:
        if _camera_lib is not None:
            raise AicbError(status, "camera construction failed")
        _check(status)


def _check(status: int):
    if status != abi.OK:
        raise AicbError(status, load_library().aicb_last_error().decode("utf-8", "replace"))


# ------------------------------------------------------------------------------------------------
# GraphicsOptions / Viewport / Camera
# ------------------------------------------------------------------------------------------------
EXPOSURE_AUTOMATIC = "automatic"   # GraphicsOptions.exposure = ExposureOption::Automatic (graphics_options.rs:380-407)


@dataclasses.dataclass
class GraphicsOptions:
    """The pixel-affecting subset of GraphicsOptions (graphics_options.rs:28-150).
    Defaults are GraphicsOptions::default() (graphics_options.rs:251-281)."""
    fog: int = FOG_ABRUPT
    fov_y: float = 90.0
    tone_mapping: int = TONE_CLAMP
    maximum_intensity: float = math.inf
    exposure: float = 1.0  # ExposureOption::Fixed(1); or EXPOSURE_AUTOMATIC (see Camera.set_measured_exposure)
    view_distance: float = 200.0
    lighting_display: int = LIGHT_LINEAR
    transparency: int = TRANSPARENCY_VOLUMETRIC
    transparency_threshold: float = 0.5
    antialiasing_always: bool = False
    debug_pixel_cost: bool = False
    bounce_samples: int = 1  # LightingOption::Bounce { samples } (graphics_options.rs:464-467)

    @staticmethod
    def unaltered_colors() -> "GraphicsOptions":
        """GraphicsOptions::UNALTERED_COLORS (graphics_options.rs:168-190)."""
        return GraphicsOptions(fog=FOG_NONE, lighting_display=LIGHT_NONE)

    def repair(self) -> "GraphicsOptions":
        """graphics_options.rs:194-198"""
        return dataclasses.replace(self, fov_y=min(max(self.fov_y, 1.0), 189.0),
                                   view_distance=min(max(self.view_distance, 1.0), 10000.0))

    def to_abi(self, include_sky: bool = True) -> abi.Options:
        o = abi.Options()
        o.fog = self.fog
        o.lighting_display = self.lighting_display
        o.transparency = self.transparency
        o.antialiasing_always = 1 if self.antialiasing_always else 0
        o.tone_mapping = self.tone_mapping
        o.debug_pixel_cost = 1 if self.debug_pixel_cost else 0
        o.include_sky = 1 if include_sky else 0
        o.bounce_samples = self.bounce_samples if self.lighting_display == LIGHT_BOUNCE else 0
        o.transparency_threshold = self.transparency_threshold
        o.maximum_intensity = self.maximum_intensity
        o.view_distance = min(max(self.view_distance, 1.0), 10000.0)
        return o


@dataclasses.dataclass
class Viewport:
    """camera/viewport.rs:24-37"""
    nominal_size: tuple
    framebuffer_size: tuple

    @staticmethod
    def with_scale(scale: float, framebuffer_size) -> "Viewport":
        w, h = framebuffer_size
        return Viewport((w / scale if scale else math.inf, h / scale if scale else math.inf), (int(w), int(h)))


class Camera:
    """Camera (camera_struct.rs:43): options + viewport + view transform -> matrices.
    Matrix construction happens in the C ABI (host code, aicb_camera_*)."""

    def __init__(self, options: GraphicsOptions, viewport: Viewport):
        self.options = options.repair()
        self.viewport = viewport
        self._rotation = (0.0, 0.0, 0.0, 1.0)
        self._translation = (0.0, 0.0, 0.0)
        # Camera::exposure_value: ExposureOption::initial(), 1 under Automatic
        self.exposure_value = 1.0 if self.options.exposure == EXPOSURE_AUTOMATIC else self.options.exposure
        self.data = abi.CameraData()
        self._compute()

    def _compute(self):
        q = (C.c_double * 4)(*self._rotation)
        t = (C.c_double * 3)(*self._translation)
        _check_cam(_cam("camera_from_view")(q, t, self.options.fov_y, self.options.view_distance,
                                         float(self.viewport.nominal_size[0]), float(self.viewport.nominal_size[1]),
                                         self.viewport.framebuffer_size[0], self.viewport.framebuffer_size[1],
                                         self.exposure_value, C.byref(self.data)))

    def set_view_transform(self, rotation_ijkr: Sequence[float], translation: Sequence[float]):
        self._rotation = tuple(float(v) for v in rotation_ijkr)
        self._translation = tuple(float(v) for v in translation)
        self._compute()

    def look_at_y_up(self, eye: Sequence[float], target: Sequence[float]):
        """camera_struct.rs:459-471"""
        e = (C.c_double * 3)(*[float(v) for v in eye])
        t = (C.c_double * 3)(*[float(v) for v in target])
        _check_cam(_cam("camera_look_at")(e, t, self.options.fov_y, self.options.view_distance,
                                       float(self.viewport.nominal_size[0]), float(self.viewport.nominal_size[1]),
                                       self.viewport.framebuffer_size[0], self.viewport.framebuffer_size[1],
                                       self.exposure_value, C.byref(self.data)))

    def set_measured_exposure(self, value: float):
        """Camera::set_measured_exposure (camera_struct.rs:169-181): with EXPOSURE_AUTOMATIC the camera's exposure
        becomes `value` (1 under LIGHT_NONE), if it is a non-negative, non-NaN f32 (PositiveSign::try_from, a zero
        of either sign being +0); a Fixed exposure ignores it.  Typically a step_exposure result."""
        v = float(np.float32(value))
        if math.isnan(v) or v < 0.0 or self.options.exposure != EXPOSURE_AUTOMATIC:
            return
        self.exposure_value = 1.0 if self.options.lighting_display == LIGHT_NONE else abs(v)
        self.data.exposure = self.exposure_value

    def project_ndc_into_world(self, x: float, y: float) -> np.ndarray:
        """camera_struct.rs:238-257 -> [ox,oy,oz,dx,dy,dz]"""
        out = (C.c_double * 6)()
        _cam("camera_project_ndc")(C.byref(self.data), x, y, out)
        return np.array(out[:], dtype=np.float64)

    NEAR_PLANE_DISTANCE = 1.0 / 32.0   # camera_struct.rs:202-205

    def projection_matrix(self) -> np.ndarray:
        """Camera::projection_matrix (camera_struct.rs:387-416): m11..m44 as a [4, 4] array, row-vector convention,
        built as host/camera.cpp builds it."""
        o = self.options
        fov_cot = 1.0 / math.tan((o.fov_y / 2.0) * (math.pi / 180.0))
        w, h = (float(v) for v in self.viewport.nominal_size)
        aspect = w / h if h != 0.0 else math.inf
        if not math.isfinite(aspect):
            aspect = 1.0
        near, far = self.NEAR_PLANE_DISTANCE, min(max(o.view_distance, 1.0), 10000.0)
        m = np.zeros((4, 4), dtype=np.float64)
        m[0, 0] = fov_cot / aspect
        m[1, 1] = fov_cot
        m[2, 2] = far / (near - far)
        m[2, 3] = -1.0
        m[3, 2] = (far * near) / (near - far)
        return m

    def depth_transform(self) -> np.ndarray:
        """The matrix RaytraceToTexture maps a ray's depth with (raytrace_to_texture.rs:613-618):
        projection_matrix().pre_translate((0, 0, -near)).pre_scale(0, 0, -(view_distance - near)), composed as euclid
        0.22 defines pre_translate (Transform3D::translation(v).then(self)) and pre_scale (rows 1-3 scaled), in f64 and
        in euclid's term order.  Returns m11..m44 as a [4, 4] array."""
        p = [[float(v) for v in row] for row in self.projection_matrix()]
        near = self.NEAR_PLANE_DISTANCE
        far = min(max(self.options.view_distance, 1.0), 10000.0)
        t = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, -near, 1.0]]
        # Transform3D::then: self.mi1 * other.m1j + self.mi2 * other.m2j + self.mi3 * other.m3j + self.mi4 * other.m4j
        m = [[t[i][0] * p[0][j] + t[i][1] * p[1][j] + t[i][2] * p[2][j] + t[i][3] * p[3][j] for j in range(4)]
             for i in range(4)]
        scale = (0.0, 0.0, -(far - near))
        for i in range(3):
            m[i] = [v * scale[i] for v in m[i]]
        return np.array(m, dtype=np.float64)

    @property
    def inverse_projection_view(self) -> np.ndarray:
        return np.array(self.data.inverse_projection_view[:], dtype=np.float64).reshape(4, 4)


def eye_for_look_at(bounds_lower, bounds_size, direction) -> np.ndarray:
    """all-is-cubes/src/camera.rs:34-40"""
    b = abi.Aab()
    b.lower[:] = [int(v) for v in bounds_lower]
    b.size[:] = [int(v) for v in bounds_size]
    d = (C.c_double * 3)(*[float(v) for v in direction])
    out = (C.c_double * 3)()
    _cam("eye_for_look_at")(C.byref(b), d, out)
    return np.array(out[:], dtype=np.float64)


# ------------------------------------------------------------------------------------------------
# Flattened Space snapshot
# ------------------------------------------------------------------------------------------------
class Block:
    """One Space palette entry as the raytracer sees it (TracingBlock, sr.rs:569-587)."""

    def __init__(self, *, color=None, emission=(0.0, 0.0, 0.0), is_air=False, resolution=1, voxel_lower=None,
                 indices: Optional[np.ndarray] = None, palette: Optional[np.ndarray] = None, selectable=True,
                 voxel_selectable=None, collision=True, voxel_collision=None):
        """selectable: BlockAttributes::selectable (AICB_BLOCK_NOT_SELECTABLE when false; an air block is never
        selectable).  voxel_selectable: each palette entry's Evoxel::selectable (a bool or a bool per entry), written
        into the palette's column 7 as AICB_VOXEL_NOT_SELECTABLE; None keeps the column as given (zero: selectable).
        collision: a single voxel's Evoxel::collision, True for BlockCollision::Hard, False for None.  voxel_collision:
        each palette entry's, a bool or a bool per entry.  Both are kept beside the palette (voxel_no_collision) and
        add AICB_VOXEL_NO_COLLISION to the flags of column 7 when the block is described to the library, so column 7
        keeps what the caller wrote there (a caller may also set the bit in it directly).  The block's own collision is
        derived from its voxels when it is placed."""
        self.is_air = bool(is_air)
        self.selectable = bool(selectable) and not self.is_air
        self.resolution = int(resolution)
        if indices is None:
            c = (0.0, 0.0, 0.0, 0.0) if color is None else tuple(color)
            self.palette = np.zeros((1, 8), dtype=np.float32)
            self.palette[0, :4] = c
            self.palette[0, 4:7] = emission
            self.indices = None
            self.voxel_lower = (0, 0, 0)
            self.voxel_size = (1, 1, 1)
            self.resolution = 1
        else:
            assert indices.ndim == 3 and indices.dtype == np.uint16
            self.indices = np.ascontiguousarray(indices)
            self.palette = np.ascontiguousarray(palette, dtype=np.float32)
            assert self.palette.ndim == 2 and self.palette.shape[1] == 8
            self.voxel_lower = tuple(int(v) for v in (voxel_lower or (0, 0, 0)))
            self.voxel_size = tuple(int(v) for v in indices.shape)
        if voxel_selectable is not None:
            if self.indices is not None and palette is not None and np.shares_memory(self.palette, palette):
                self.palette = self.palette.copy()
            sel = np.broadcast_to(np.asarray(voxel_selectable, dtype=bool), (self.palette.shape[0],))
            self.palette.view(np.uint32)[:, 7] = np.where(sel, 0, abi.VOXEL_NOT_SELECTABLE).astype(np.uint32)
        if self.indices is None and not collision:
            voxel_collision = False
        self.voxel_no_collision = None if voxel_collision is None else ~np.broadcast_to(
            np.asarray(voxel_collision, dtype=bool), (self.palette.shape[0],)).copy()
        self._derive_for_light()

    def desc_palette(self) -> np.ndarray:
        """The palette as the library reads it: column 7 with AICB_VOXEL_NO_COLLISION added where voxel_no_collision
        says so (the palette itself when it says nothing)."""
        mask = getattr(self, "voxel_no_collision", None)
        if mask is None or not mask.any():
            return self.palette
        pal = np.array(self.palette, dtype=np.float32, copy=True)
        col = pal.view(np.uint32)[:, 7]
        col[mask] |= np.uint32(abi.VOXEL_NO_COLLISION)
        return pal

    def _derive_for_light(self):
        """EvaluatedBlock derived data read by light propagation (block/eval/derived.rs:80-104 for single voxels,
        :105-235 for recursive blocks: a restatement for the synthetic blocks of the tests and benches — block
        evaluation itself is out of scope, SURVEY §2 #11; the oracle and the GPU consume whatever is supplied here)."""
        if self.is_air:
            self.light_opaque_faces = 0
            self.light_visible = False
            self.light_color = (0.0, 0.0, 0.0, 0.0)
            self.light_face_colors = [(0.0, 0.0, 0.0, 0.0)] * 6
            self.light_emission = (0.0, 0.0, 0.0)
            return
        if self.indices is None:
            c = tuple(float(v) for v in self.palette[0, :4])
            e = tuple(float(v) for v in self.palette[0, 4:7])
            self.light_color = c
            self.light_face_colors = [c] * 6
            self.light_emission = e
            self.light_opaque_faces = 0x3F if c[3] == 1.0 else 0
            self.light_visible = (c[3] != 0.0) or any(v != 0.0 for v in e)
            return
        # compute_derived (block/eval/derived.rs:80-235): every face is "rendered" by axis-aligned rays through the voxel
        # data (trace_for_eval, raytracer_components.rs:174-200), starting at the first layer of the DATA bounds seen
        # from that face; a face colour is the alpha-weighted mean of its pixels with alpha = coverage of the full
        # face.  The sums run in numpy's order, not iproduct!'s: last-bit differences only.
        f32 = np.float32
        r = self.resolution
        lo, sz = self.voxel_lower, self.voxel_size
        vox = self.palette[self.indices]            # [sx, sy, sz, 8]: rgba, emission
        thickness = f32(1.0) / f32(r)

        # apply_transmittance (raytracer_components.rs:215-258) of every voxel for thickness 1/resolution
        alpha_v = vox[..., 3]
        unit_t = (f32(1.0) - alpha_v).astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore"):
            depth_t = np.power(unit_t, thickness, dtype=np.float32)
            adj = np.clip(f32(1.0) - depth_t, f32(0.0), f32(1.0)).astype(np.float32)
            coeff = np.where(unit_t == 1.0, thickness, np.maximum((depth_t - f32(1.0)) / (unit_t - f32(1.0)), f32(0.0))).astype(np.float32)
        adj = np.where(alpha_v >= 1.0, f32(1.0), np.where(alpha_v <= 0.0, f32(0.0), adj)).astype(np.float32)
        coeff = np.where(alpha_v >= 1.0, f32(1.0), coeff).astype(np.float32)

        self.light_opaque_faces = 0
        cols = []
        all_color = np.zeros(3, dtype=np.float32)
        all_alpha = f32(0.0)
        all_em = np.zeros(3, dtype=np.float32)
        count = 0
        area = f32(r * r)
        for f in range(6):                          # NX NY NZ PX PY PZ
            axis, positive = f % 3, f >= 3
            # trace_for_eval for all pixels of the face at once: layers of the data from the face inwards
            order = range(sz[axis] - 1, -1, -1) if positive else range(sz[axis])
            shape = tuple(sz[a] for a in range(3) if a != axis)
            light = np.zeros(shape + (3,), dtype=np.float32)
            T = np.ones(shape, dtype=np.float32)
            em = np.zeros(shape + (3,), dtype=np.float32)
            live = np.ones(shape, dtype=bool)
            for k in order:
                v = np.take(vox, k, axis=axis)
                a = np.take(adj, k, axis=axis)
                c = np.take(coeff, k, axis=axis)
                em = np.where(live[..., None], em + (v[..., 4:7] * c[..., None]) * T[..., None], em).astype(np.float32)
                light = np.where(live[..., None], light + (v[..., :3] * a[..., None]) * T[..., None], light).astype(np.float32)
                T = np.where(live, T * (f32(1.0) - a), T).astype(np.float32)
                live &= ~(T < f32(1.0 / 256.0))
                if not live.any():
                    break
            pa = np.where(T >= 1.0, f32(0.0), f32(1.0) - T).astype(np.float32)              # Rgba::from(ColorBuf)
            with np.errstate(invalid="ignore", divide="ignore"):
                prgb = np.where(pa[..., None] > 0, light / pa[..., None], f32(0.0)).astype(np.float32)
            csum = (prgb * pa[..., None]).reshape(-1, 3).sum(axis=0, dtype=np.float32)
            asum = f32(pa.sum(dtype=np.float32))
            all_em = (all_em + em.reshape(-1, 3).sum(axis=0, dtype=np.float32)).astype(np.float32)
            count += pa.size
            all_color = (all_color + csum).astype(np.float32)
            all_alpha = f32(all_alpha + asum)
            if asum > 0:
                cm = csum / asum
                cols.append((float(cm[0]), float(cm[1]), float(cm[2]), float(min(max(asum / area, f32(0.0)), f32(1.0)))))
            else:
                cols.append((0.0, 0.0, 0.0, 0.0))
            # opaque[face] (derived.rs:196-209): the block's own surface layer lies inside the data and is fully opaque
            others = [a_ for a_ in range(3) if a_ != axis]
            covers = all((lo[a_] == 0 and sz[a_] == r) for a_ in others) and \
                ((lo[axis] + sz[axis] == r) if positive else (lo[axis] == 0))
            if covers and np.all(np.take(alpha_v, sz[axis] - 1 if positive else 0, axis=axis) == 1.0):
                self.light_opaque_faces |= 1 << f
        self.light_face_colors = cols
        surface = f32(6 * r * r)
        if all_alpha > 0:
            c = all_color / all_alpha
            self.light_color = (float(c[0]), float(c[1]), float(c[2]), float(min(max(all_alpha / surface, f32(0.0)), f32(1.0))))
        else:
            self.light_color = (0.0, 0.0, 0.0, 0.0)
        self.light_emission = tuple(float(v) for v in (all_em / surface)) if count else (0.0, 0.0, 0.0)
        self.light_visible = bool((vox[..., 3] != 0).any() or (vox[..., 4:7] != 0).any())

    def set_light_data(self, bl: "BlockLight"):
        """Take compute_derived's light fields (Context.derive_block_light) in place of the numpy restatement."""
        self.light_face_colors = list(bl.face_colors)
        self.light_color = bl.color
        self.light_emission = bl.emission
        self.light_opaque_faces = bl.opaque_faces
        self.light_visible = bl.visible

    @staticmethod
    def air() -> "Block":
        return Block(is_air=True)


@dataclasses.dataclass(frozen=True)
class BlockLight:
    """compute_derived's light fields of one block (block/eval/derived.rs:80-216): the face colours NX..PZ, colour and
    emission, the faces opaque to light (bit face - 1) and Derived::visible."""
    face_colors: tuple
    color: tuple
    emission: tuple
    opaque_faces: int
    visible: bool

    @staticmethod
    def from_abi(o: abi.BlockLight) -> "BlockLight":
        return BlockLight(face_colors=tuple(tuple(o.face_colors[f][:]) for f in range(6)), color=tuple(o.color[:]),
                          emission=tuple(o.emission[:]), opaque_faces=int(o.opaque_faces), visible=bool(o.visible))


class DeviceBlock:
    """A block definition whose voxels are CUDA tensors on the scene's device (device 0 of a group), for
    update_blocks / append_blocks (aicb_scene_*_blocks_device): `indices` a uint16 tensor of the data bounds' shape
    (Z-major), or None for a single voxel, palette[0]; `palette` a float32 [n, 8] tensor (rgba, emission, pad).
    `light` is the block's BlockLight, or None to derive it on the device (AICB_BLOCKS_DERIVE_LIGHT); `visible`
    ORs an animation hint into a derived Derived::visible.  Column 7 of the palette holds each voxel's flags as the
    bits of the float32 (AICB_VOXEL_NOT_SELECTABLE); `selectable` is BlockAttributes::selectable."""

    def __init__(self, resolution, voxel_lower, indices, palette, is_air=False, light: Optional["BlockLight"] = None,
                 visible: bool = False, selectable: bool = True):
        self.selectable = bool(selectable)
        self.resolution = int(resolution)
        self.voxel_lower = tuple(int(v) for v in (voxel_lower or (0, 0, 0)))
        self.indices = indices
        self.palette = palette
        self.is_air = bool(is_air)
        self.light = light
        self.visible = bool(visible)

    def _check(self, device):
        torch = _torch()
        for name, t, dtype in (("indices", self.indices, torch.uint16), ("palette", self.palette, torch.float32)):
            if t is None and name == "indices":
                continue
            if not _is_cuda_tensor(t) or t.dtype != dtype or t.device != device or not t.is_contiguous():
                raise ValueError(f"DeviceBlock.{name} must be a contiguous {dtype} tensor on {device}")
        if self.palette.dim() != 2 or self.palette.shape[1] != 8:
            raise ValueError("DeviceBlock.palette must have shape [n, 8]")
        if self.indices is not None and self.indices.dim() != 3:
            raise ValueError("DeviceBlock.indices must have 3 dimensions (the data bounds)")

    def fill_desc(self, bd):
        """DeviceBlock -> aicb_block_desc with device pointers (the tensors stay owned by the block)."""
        bd.resolution = 1 if self.indices is None else self.resolution
        bd.is_air = 1 if self.is_air else 0
        bd.voxel_bounds.lower[:] = (0, 0, 0) if self.indices is None else self.voxel_lower
        bd.voxel_bounds.size[:] = (1, 1, 1) if self.indices is None else tuple(self.indices.shape)
        bd.indices = None if self.indices is None else self.indices.data_ptr()
        bd.n_indices = 0 if self.indices is None else self.indices.numel()
        bd.palette = self.palette.data_ptr() if self.palette.shape[0] else None
        bd.n_palette = self.palette.shape[0]
        bd.flags = 0 if self.selectable else abi.BLOCK_NOT_SELECTABLE
        bl = self.light
        if bl is None:
            bd.light_visible = 1 if self.visible else 0
            return
        bd.light_opaque_faces = bl.opaque_faces
        bd.light_visible = 1 if bl.visible else 0
        for f in range(6):
            bd.light_face_colors[f][:] = bl.face_colors[f]
        bd.light_color[:] = bl.color
        bd.light_emission[:] = bl.emission


def exposure_states(n):
    """n default exposure::State values (exposure.rs:50-58): every sample 1.0, index 0, log 0; an
    abi.EXPOSURE_STATE_DTYPE array."""
    st = np.zeros(n, dtype=abi.EXPOSURE_STATE_DTYPE)
    st["luminance_samples"] = 1.0
    return st


def view_transform_matrix(rotation_ijkr, translation) -> np.ndarray:
    """ViewTransform::to_transform of an eye's view transform (aicb_view_transform_matrix): the eye-to-world matrix
    step_exposure takes, m11..m44 as 16 float64 in the row-vector convention of Camera."""
    q = (C.c_double * 4)(*[float(v) for v in rotation_ijkr])
    t = (C.c_double * 3)(*[float(v) for v in translation])
    out = (C.c_double * 16)()
    load_library().aicb_view_transform_matrix(q, t, out)
    return np.array(out[:], dtype=np.float64)


def eyes(n):
    """n CharacterEye::default() values with no previous velocity: an abi.EYE_DTYPE array of zeros."""
    return np.zeros(n, dtype=abi.EYE_DTYPE)


def look_rotation(yaw_degrees: float, pitch_degrees: float) -> np.ndarray:
    """Body::look_rotation (physics/body.rs:285-292) of a yaw and a pitch in degrees: the eye-to-world rotation
    (i, j, k, r) as float64 [4], what eye_views takes per eye."""
    out = (C.c_double * 4)()
    load_library().aicb_look_rotation(float(yaw_degrees), float(pitch_degrees), out)
    return np.array(out[:], dtype=np.float64)


def eye_view_params(options: "GraphicsOptions", viewport: "Viewport") -> abi.EyeViewParams:
    """The aicb_eye_view_params of a batch of eyes whose world cameras have these options and this viewport."""
    o = options.repair()
    p = abi.EyeViewParams()
    p.fov_y_degrees = o.fov_y
    p.view_distance = o.view_distance
    p.nominal_width = float(viewport.nominal_size[0])
    p.nominal_height = float(viewport.nominal_size[1])
    p.fb_width, p.fb_height = (int(v) for v in viewport.framebuffer_size)
    automatic = o.exposure == EXPOSURE_AUTOMATIC
    p.fixed_exposure = 1.0 if automatic else float(o.exposure)
    p.automatic_exposure = 1 if automatic else 0
    p.lighting_display = o.lighting_display
    return p


def eye_cameras(n, options: "GraphicsOptions", viewport: "Viewport") -> np.ndarray:
    """A camera table of n world cameras as Camera::new leaves them (identity view transform, exposure
    ExposureOption::initial()): the abi.CAMERA_DTYPE array eye_views updates in place."""
    cam = Camera(options, viewport)
    return np.repeat(np.frombuffer(bytes(cam.data), dtype=abi.CAMERA_DTYPE), n)


def bodies(n, position=(0.0, 0.0, 0.0), collision_box=(-0.5, -0.5, -0.5, 0.5, 0.5, 0.5), velocity=(0.0, 0.0, 0.0),
           flying=False, noclip=False):
    """n bodies as Body::new_minimal makes them (occupying: the box at the position), an abi.BODY_DTYPE array.  Each
    argument is one value or one per body."""
    b = np.zeros(n, dtype=abi.BODY_DTYPE)
    p = np.broadcast_to(np.asarray(position, dtype=np.float64), (n, 3))
    box = np.broadcast_to(np.asarray(collision_box, dtype=np.float64), (n, 6))
    b["position"] = p
    b["velocity"] = np.broadcast_to(np.asarray(velocity, dtype=np.float64), (n, 3))
    b["collision_box"] = box
    b["occupying"][:, :3] = box[:, :3] + p
    b["occupying"][:, 3:] = box[:, 3:] + p
    b["flying"] = flying
    b["noclip"] = noclip
    return b


class Space:
    """What SpaceRaytracer::new reads from space::Read (sr.rs:64-88): bounds, per-cube block
    index (shape [X,Y,Z], C order == Vol Z-major, vol.rs:1013-1018), optional PackedLight texels
    (shape [X,Y,Z,4]), block table, sky."""

    def __init__(self, lower, block_ids: np.ndarray, blocks: Sequence[Block], light: Optional[np.ndarray] = None,
                 sky_colors=None, light_max_distance: int = 0):
        assert block_ids.ndim == 3
        self.lower = tuple(int(v) for v in lower)
        self.block_ids = np.ascontiguousarray(block_ids, dtype=np.uint16)
        self.size = tuple(int(v) for v in self.block_ids.shape)
        self.blocks = list(blocks)
        self.light = None if light is None else np.ascontiguousarray(light, dtype=np.uint8)
        if self.light is not None:
            assert self.light.shape == self.size + (4,)
        if sky_colors is None:
            # Sky::DEFAULT = Uniform(DAY_SKY_COLOR = srgb[243 243 255]) (sky.rs:24, palette.rs:63)
            sky_colors = [srgb8_to_linear((243, 243, 255))]
        self.sky_colors = _sky_colors(sky_colors)
        self.light_max_distance = int(light_max_distance)

    def to_desc(self):
        """Returns (abi.SceneDesc, keepalive list)."""
        keep = []
        d = abi.SceneDesc()
        d.bounds.lower[:] = self.lower
        d.bounds.size[:] = self.size
        d.block_ids = self.block_ids.ctypes.data
        d.light = self.light.ctypes.data if self.light is not None else None
        arr = (abi.BlockDesc * len(self.blocks))()
        for i, b in enumerate(self.blocks):
            fill_block_desc(arr[i], b)
            keep.append(b)
        d.blocks = arr
        d.n_blocks = len(self.blocks)
        d.sky = _sky(self.sky_colors)
        d.light_max_distance = self.light_max_distance
        keep.append(arr)
        keep.append(self)
        return d, keep


class DeviceSpace:
    """Space's device twin, as DeviceBlock is Block's, for a world that lives on the GPU: SpaceRaytracer, GroupScene,
    DeviceGroup.add_scene / update and RtRenderer.update create the scene from it on the device
    (aicb_scene_create_device), on the device's current torch stream.  `block_ids` is a contiguous uint16 CUDA tensor
    [X, Y, Z] (Z-major); `light` a contiguous uint8 tensor [X, Y, Z, 4] on the same device, or None; `blocks` are
    DeviceBlocks whose light is given for all of them, or derived on the device for all (light=None).  The tensors
    must stay unchanged until the scene is created; the scene does not keep them."""

    def __init__(self, lower, block_ids, blocks: Sequence["DeviceBlock"], light=None, sky_colors=None,
                 light_max_distance: int = 0):
        torch = _torch()
        if (not _is_cuda_tensor(block_ids) or block_ids.dtype != torch.uint16 or block_ids.dim() != 3
                or not block_ids.is_contiguous()):
            raise ValueError("DeviceSpace.block_ids must be a contiguous uint16 CUDA tensor [X, Y, Z]")
        self.device = block_ids.device
        self.lower = tuple(int(v) for v in lower)
        self.block_ids = block_ids
        self.size = tuple(int(v) for v in block_ids.shape)
        if light is not None and (not _is_cuda_tensor(light) or light.dtype != torch.uint8 or light.device != self.device
                                  or tuple(light.shape) != self.size + (4,) or not light.is_contiguous()):
            raise ValueError(f"DeviceSpace.light must be a contiguous uint8 tensor {list(self.size) + [4]} on "
                             f"{self.device}, or None")
        self.light = light
        self.blocks = list(blocks)
        if not all(isinstance(b, DeviceBlock) for b in self.blocks):
            raise ValueError("DeviceSpace.blocks must all be DeviceBlocks")
        derive = [b.light is None for b in self.blocks]
        if any(derive) and not all(derive):
            raise ValueError("a DeviceSpace derives the light of every block (light=None) or of none")
        for b in self.blocks:
            b._check(self.device)
        self.flags = abi.BLOCKS_DERIVE_LIGHT if any(derive) else 0
        if sky_colors is None:
            sky_colors = [srgb8_to_linear((243, 243, 255))]
        self.sky_colors = _sky_colors(sky_colors)
        self.light_max_distance = int(light_max_distance)

    def to_desc(self, device):
        """Returns (abi.SceneDesc with device pointers, keepalive list); ValueError unless the tensors are on
        `device`."""
        if self.device != device:
            raise ValueError(f"the DeviceSpace's tensors are on {self.device}, the scene's device is {device}")
        d = abi.SceneDesc()
        d.bounds.lower[:] = self.lower
        d.bounds.size[:] = self.size
        d.block_ids = self.block_ids.data_ptr()
        d.light = self.light.data_ptr() if self.light is not None else None
        arr = (abi.BlockDesc * max(len(self.blocks), 1))()
        for i, b in enumerate(self.blocks):
            b.fill_desc(arr[i])
        d.blocks = arr
        d.n_blocks = len(self.blocks)
        d.sky = _sky(self.sky_colors)
        d.light_max_distance = self.light_max_distance
        return d, [arr, self]


def _create_scene(fn, owner, space, device, out):
    """aicb_scene_create or aicb_group_scene_create (`fn`) on `owner`; a DeviceSpace through their device form on the
    device's current torch stream."""
    lib = load_library()
    if isinstance(space, DeviceSpace):
        desc, keep = space.to_desc(device)
        _check(getattr(lib, fn + "_device")(owner, C.byref(desc), space.flags, _stream(device), C.byref(out)))
    else:
        desc, keep = space.to_desc()
        _check(getattr(lib, fn)(owner, C.byref(desc), C.byref(out)))
    del keep


def _sky_colors(sky_colors) -> np.ndarray:
    """One row: Sky::Uniform; eight rows: Sky::Octants (index (x>=0)<<2 | (y>=0)<<1 | (z>=0))."""
    c = np.asarray(sky_colors, dtype=np.float32).reshape(-1, 3)
    assert c.shape[0] in (1, 8)
    return c


def _sky(sky_colors) -> abi.Sky:
    c = _sky_colors(sky_colors)
    sky = abi.Sky()
    sky.kind = 0 if c.shape[0] == 1 else 1
    for k in range(c.shape[0]):
        sky.colors[k][:] = [float(v) for v in c[k]]
    return sky


def fill_block_desc(bd, b):
    """Block -> aicb_block_desc (the arrays stay owned by `b`)."""
    bd.resolution = b.resolution
    bd.is_air = 1 if b.is_air else 0
    bd.voxel_bounds.lower[:] = b.voxel_lower
    bd.voxel_bounds.size[:] = b.voxel_size
    if b.indices is not None:
        bd.indices = b.indices.ctypes.data
        bd.n_indices = b.indices.size
    else:
        bd.indices = None
        bd.n_indices = 0
    pal = b.desc_palette() if hasattr(b, "desc_palette") else b.palette
    b._desc_palette = pal   # kept alive with the block, which the caller keeps
    bd.palette = pal.ctypes.data
    bd.n_palette = pal.shape[0]
    bd.light_opaque_faces = b.light_opaque_faces
    bd.light_visible = 1 if b.light_visible else 0
    for f in range(6):
        bd.light_face_colors[f][:] = b.light_face_colors[f]
    bd.light_color[:] = b.light_color
    bd.light_emission[:] = b.light_emission
    bd.flags = 0 if getattr(b, "selectable", True) else abi.BLOCK_NOT_SELECTABLE


def _block_descs(blocks):
    """Blocks -> an aicb_block_desc array (its arrays stay owned by the blocks)."""
    arr = (abi.BlockDesc * max(len(blocks), 1))()
    for i, b in enumerate(blocks):
        fill_block_desc(arr[i], b)
    return arr


def light_chart():
    """The static light-ray chart (space/light/chart/generator.rs) as (weights [n,6] f32, children [n,6] u32)."""
    lib = load_library()
    n = lib.aicb_light_chart(None, None)
    w = np.zeros((n, 6), dtype=np.float32)
    ch = np.zeros((n, 6), dtype=np.uint32)
    lib.aicb_light_chart(w.ctypes.data, ch.ctypes.data)
    return w, ch


def light_chart_chains():
    """The chart as the chain walk sees it: (preorder [n] -> node of light_chart(), chains [c,6] u32 = first node in
    preorder, nodes, child chains, first child chain, parent's branch slot, own branch slot; euler [2c] u16)."""
    lib = load_library()
    lib.aicb_light_chart_chains.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.aicb_light_chart_chains.restype = C.c_uint32
    n_nodes = lib.aicb_light_chart(None, None)
    n_chains = lib.aicb_light_chart_chains(None, None, None)
    pre = np.zeros(n_nodes, dtype=np.uint32)
    chains = np.zeros((n_chains, 6), dtype=np.uint32)
    euler = np.zeros(2 * n_chains, dtype=np.uint16)
    lib.aicb_light_chart_chains(pre.ctypes.data, chains.ctypes.data, euler.ctypes.data)
    return pre, chains, euler


def srgb8_to_linear(rgb) -> tuple:
    """component_from_srgb8 (color.rs): f32 sRGB decode, used only for named palette constants."""
    out = []
    for c in rgb:
        f = np.float32(c) / np.float32(255.0)
        if f <= np.float32(0.04045):
            out.append(float(np.float32(f * np.float32(25.0 / 323.0))))
        else:
            x = np.float32(np.float32(200.0) * f + np.float32(11.0)) / np.float32(211.0)
            out.append(float(np.float32(float(x) ** float(np.float32(12.0 / 5.0)))))
    return tuple(out)


# ------------------------------------------------------------------------------------------------
# SpaceRaytracer / RtRenderer
# ------------------------------------------------------------------------------------------------
class Context:
    _default = None

    def __init__(self, device_id: int = -1):
        lib = load_library()
        self.handle = C.c_void_p()
        _check(lib.aicb_ctx_create(device_id, C.byref(self.handle)))
        self.device_id = lib.aicb_ctx_device(self.handle)   # -1 resolved to the device current at creation
        self._pending = None   # the DeviceRendering issued last and not finished yet

    def settle(self):
        """Finish the asynchronous call issued last on this context, if it is not finished yet: the context tracks one
        frame, so its next render call, or a change of one of its scenes, must come after that call's finish."""
        if self._pending is not None:
            self._pending.result()

    @classmethod
    def default(cls) -> "Context":
        if cls._default is None:
            cls._default = Context(-1)
        return cls._default

    def derive_block_light(self, blocks: Sequence[Block]) -> list:
        """compute_derived's light fields of every block on this context's device (aicb_derive_block_light), one
        BlockLight per block.  Raises AicbError (ERR_INVALID) for a block scene creation rejects, or where the
        reference's colour or emission sum is NaN and it panics."""
        if not blocks:
            return []
        descs = _block_descs(blocks)
        out = (abi.BlockLight * len(blocks))()
        _check(load_library().aicb_derive_block_light(self.handle, descs, len(blocks), out))
        return [BlockLight.from_abi(o) for o in out]

    def close(self):
        if self.handle:
            load_library().aicb_ctx_destroy(self.handle)
            self.handle = C.c_void_p()


@dataclasses.dataclass
class RenderInfo:
    cubes_traced: int
    rays: int
    algorithmic_bytes: int
    counters: tuple
    kernel_ms: float
    flaws: int
    # first chunk: ray generation, marching, shading, encode; where shading and encode ran as one kernel
    # (resolve_kernel: None / Flat lighting, most frames) [2] is its time and [3] is 0
    stage_ms: tuple = (0.0, 0.0, 0.0, 0.0)
    # 1: the rays were taken in order of their tiles' steps in the context's previous frame of the same view and layout;
    # 0: by chord
    ray_order: int = 0

    @staticmethod
    def from_abi(i: abi.RenderInfo) -> "RenderInfo":
        return RenderInfo(int(i.cubes_traced), int(i.rays), int(i.algorithmic_bytes), tuple(int(c) for c in i.counters),
                          float(i.kernel_ms), int(i.flaws), tuple(float(v) for v in i.stage_ms), int(i.ray_order))


@dataclasses.dataclass
class Rendering:
    """headless.rs:52-67"""
    size: tuple
    data: np.ndarray  # [H, W, 4] uint8 sRGB RGBA
    flaws: int
    info: RenderInfo


# ------------------------------------------------------------------------------------------------
# outputs in device memory (aicb_device_outputs): torch tensors, issued on torch.cuda.current_stream()
# ------------------------------------------------------------------------------------------------
def _torch():
    import torch
    return torch


def _ctx_device(ctx: "Context"):
    return _torch().device("cuda", ctx.device_id)


def _device_outputs(out, device, spec) -> dict:
    """The output tensors of a device call: spec maps a name to (shape, dtype); `out` (a tensor for a call of one output,
    or a dict of them) supplies the caller's own tensors, checked for shape, dtype, device and contiguity; the others
    are allocated with torch's caching allocator."""
    torch = _torch()
    given = out if isinstance(out, dict) else ({next(iter(spec)): out} if out is not None else {})
    unknown = set(given) - set(spec)
    if unknown:
        raise ValueError(f"out= names outputs this call does not make: {sorted(unknown)}")
    tensors = {}
    for name, (shape, dtype) in spec.items():
        t = given.get(name)
        if t is None:
            t = torch.empty(shape, dtype=dtype, device=device)
        elif tuple(t.shape) != tuple(shape) or t.dtype != dtype or t.device != device or not t.is_contiguous():
            raise ValueError(f"out[{name!r}] must be a contiguous {dtype} tensor of shape {tuple(shape)} on {device}, "
                             f"not {t.dtype} {tuple(t.shape)} on {t.device}")
        tensors[name] = t
    return tensors


def _outs_abi(n: int, tensors: dict) -> abi.DeviceOutputs:
    o = abi.DeviceOutputs()
    for name, t in tensors.items():
        setattr(o, name, t.data_ptr())
    o.len = n
    return o


def _stream(device) -> int:
    """The current torch stream of `device` as a cudaStream_t.  torch's default stream is the legacy default stream:
    it goes as cudaStreamLegacy (1), since NULL names the context's own stream."""
    return _torch().cuda.current_stream(device).cuda_stream or 1


class DeviceRendering:
    """A device-output call issued on one context (device=True): its outputs are torch tensors on the scene's device,
    written in the order of the stream that was current when it was issued; nothing has synchronised.  result()
    finishes the call (aicb_render_finish: the host waits for the frame), re-issues it into the same tensors on the same
    stream when its hit stream overflowed, and returns what the host call returns, with tensors in place of arrays;
    `info` is then the call's RenderInfo.  The context tracks one frame: the next call on the context (a render, an
    update of one of its scenes, a light call) finishes this one first (Context.settle)."""

    def __init__(self, scene, issue, build):
        self._scene = scene      # the scene that aicb_render_finish finishes (kept alive until then)
        self._issue = issue
        self._build = build
        self._result = None
        self.info = None
        scene.ctx.settle()
        _check(issue())
        scene.ctx._pending = self

    def result(self):
        if self.info is None:
            ctx = self._scene.ctx
            if ctx._pending is self:
                ctx._pending = None
            lib = load_library()
            info = abi.RenderInfo()
            status = lib.aicb_render_finish(self._scene.handle, C.byref(info))
            while status == abi.ERR_RETRY:   # the capacity has been raised: the same call again
                _check(self._issue())
                status = lib.aicb_render_finish(self._scene.handle, C.byref(info))
            _check(status)
            self.info = RenderInfo.from_abi(info)
            self._result = self._build(self.info)
        return self._result


def _colorbuf_spec(n, want_depth, want_hit, want_steps) -> dict:
    torch = _torch()
    spec = {"colorbuf": ((n, 4), torch.float32)}
    if want_depth:
        spec["depth"] = ((n,), torch.float64)
    if want_hit:
        spec["hit"] = ((n, 8), torch.int32)
    if want_steps:
        spec["steps"] = ((n,), torch.uint32)
    return spec


def _colorbuf_result(t: dict, info) -> dict:
    return {"colorbuf": t["colorbuf"], "depth": t.get("depth"), "hit": t.get("hit"), "steps": t.get("steps"),
            "info": info}


def _terminal_result(t: dict, info) -> dict:
    """aicb_terminal_pixel as int32 [H, W, 6]: rgba (f32 bits), text, layer."""
    px = t["terminal"]
    return {"text": px[..., 4], "layer": px[..., 5], "rgba": px[..., :4].view(_torch().float32), "info": info}


class _Scene:
    """The calls SpaceRaytracer and GroupScene share: updates of the scene and light propagation.  Each calls the C
    function aicb_<name> through `_prefix` ("aicb_" on one context, "aicb_group_" on a group)."""

    _prefix = "aicb_"

    def _fn(self, name: str):
        """This kind of scene's form of the C function aicb_<name> (on a group, aicb_group_<name>), once the context's
        asynchronous call issued last is finished."""
        if hasattr(self, "ctx"):
            self.ctx.settle()
        return getattr(load_library(), self._prefix + name)

    def close(self):
        if self.handle:
            self._fn("scene_destroy")(self.handle)
            self.handle = C.c_void_p()

    # ---- arrays in device memory: a CUDA tensor where a numpy array goes, read on the device (aicb_*_device) ----
    def _tensor(self, x, dtype, shape, name):
        """x as a device call takes it: a contiguous tensor of `dtype` and `shape` on the scene's device (device 0 of a
        group); ValueError otherwise."""
        device = self._device()
        if (not _is_cuda_tensor(x) or x.dtype != dtype or x.device != device or not x.is_contiguous()
                or tuple(x.shape) != tuple(shape)):
            kind = str(dtype).replace("torch.", "")
            raise ValueError(f"{name} must be a contiguous {kind} tensor {list(shape)} on {device}")
        return x

    def _cube_list(self, cubes, block_ids, light=None):
        """A device call's cube list: int32 [n, 3] cubes, uint16 [n] ids, uint8 [n, 4] light or None."""
        torch = _torch()
        n = cubes.shape[0] if _is_cuda_tensor(cubes) and cubes.dim() == 2 else -1
        c = self._tensor(cubes, torch.int32, (n, 3), "cubes")
        ids = self._tensor(block_ids, torch.uint16, (n,), "block_ids")
        lt = None if light is None else self._tensor(light, torch.uint8, (n, 4), "light")
        return c, ids, lt, n

    def _region_device(self, lower, size, block_ids):
        """_region with the ids a uint16 tensor of shape `size` on the scene's device, or one id."""
        region = abi.Aab()
        region.lower[:] = [int(v) for v in lower]
        region.size[:] = [int(v) for v in size]
        if not _is_cuda_tensor(block_ids) and np.ndim(block_ids) == 0:
            return region, None, int(block_ids)
        return region, self._tensor(block_ids, _torch().uint16, tuple(region.size), "block_ids"), 0

    def block_ids(self, device: bool = False):
        """Each cube's block id, shaped like the Space, decoded from the scene's cells: a numpy uint16 array, or with
        device=True a uint16 tensor on the scene's device (device 0 of a group), ordered before the work queued
        afterwards on its current torch stream."""
        torch = _torch()
        dev = self._device()
        out = torch.empty(self.space.size, dtype=torch.uint16 if device else torch.int16, device=dev)
        _check(self._fn("scene_download_ids_device")(self.handle, out.data_ptr(), out.numel(), _stream(dev)))
        return out if device else out.cpu().numpy().view(np.uint16)

    def cursor_raycast(self, origin_dir, max_distance=None, device: bool = False):
        """cursor_raycast (cursor.rs:26-107) for a batch of rays [n, 6] (origin, direction): a numpy array of
        abi.CURSOR_DTYPE, block_id abi.CURSOR_NONE where nothing was selected.  max_distance: None (f64::INFINITY), a
        number or one per ray.  device=True: origin_dir (and max_distance, if an array) are float64 tensors on the
        scene's device (device 0 of a group), the call is issued on its current torch stream, and the result is a
        uint8 tensor [n, 80] (view it with .cpu().numpy().view(abi.CURSOR_DTYPE))."""
        if device:
            torch = _torch()
            dev = self._device()
            od = origin_dir.reshape(-1, 6)
            n = od.shape[0]
            od = self._tensor(od, torch.float64, (n, 6), "origin_dir")
            md = None
            if max_distance is not None:
                md = max_distance if _is_cuda_tensor(max_distance) else torch.full((n,), float(max_distance),
                                                                                   dtype=torch.float64, device=dev)
                md = self._tensor(md, torch.float64, (n,), "max_distance")
            out = torch.empty((n, 80), dtype=torch.uint8, device=dev)
            _check(self._fn("cursor_raycast_device")(self.handle, od.data_ptr(), None if md is None else md.data_ptr(),
                                                      n, out.data_ptr(), _stream(dev)))
            return out
        od = np.ascontiguousarray(origin_dir, dtype=np.float64).reshape(-1, 6)
        n = od.shape[0]
        md = None if max_distance is None else np.ascontiguousarray(np.broadcast_to(
            np.asarray(max_distance, dtype=np.float64), (n,)))
        out = np.zeros(n, dtype=abi.CURSOR_DTYPE)
        _check(self._fn("cursor_raycast")(self.handle, od.ctypes.data, None if md is None else md.ctypes.data, n,
                                          out.ctypes.data))
        return out

    def step_bodies(self, bodies, dt, gravity, external_delta_v=None, max_contacts: int = 16, device: bool = False):
        """step_one_body (physics/step.rs:316-590) against this scene for a batch of bodies: (bodies, info, contacts).
        bodies: an abi.BODY_DTYPE array (see aicb200.bodies); info: abi.BODY_STEP_INFO_DTYPE; contacts:
        abi.CONTACT_DTYPE [n, max_contacts], each body's ContactSet in first-insertion order (info["n_contacts"] of
        them, at most max_contacts).  gravity: SpacePhysics::gravity; dt: Tick::delta_t in seconds, in (0, 1];
        external_delta_v: None or [n, 3].  device=True: bodies is a uint8 CUDA tensor [n, 152] on the scene's device
        (device 0 of a group), stepped in place on its current torch stream; external_delta_v a float64 tensor [n, 3]
        or None; info and contacts are returned as uint8 tensors [n, 312] and [n, max_contacts, 28] (view them with
        .cpu().numpy().view(abi.BODY_STEP_INFO_DTYPE) etc.)."""
        g = np.ascontiguousarray(gravity, dtype=np.float64).reshape(3)
        if device:
            torch = _torch()
            dev = self._device()
            n = bodies.shape[0]
            b = self._tensor(bodies, torch.uint8, (n, abi.BODY_DTYPE.itemsize), "bodies")
            edv = None if external_delta_v is None else self._tensor(external_delta_v, torch.float64, (n, 3),
                                                                      "external_delta_v")
            info = torch.empty((n, abi.BODY_STEP_INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
            contacts = torch.zeros((n, max_contacts, abi.CONTACT_DTYPE.itemsize), dtype=torch.uint8, device=dev)
            _check(self._fn("step_bodies_device")(self.handle, b.data_ptr(), None if edv is None else edv.data_ptr(),
                                                   n, float(dt), g.ctypes.data, info.data_ptr(),
                                                   contacts.data_ptr() if max_contacts else None, max_contacts,
                                                   _stream(dev)))
            return b, info, contacts
        b = np.ascontiguousarray(bodies, dtype=abi.BODY_DTYPE).copy()
        n = b.shape[0]
        edv = None if external_delta_v is None else np.ascontiguousarray(
            np.broadcast_to(np.asarray(external_delta_v, dtype=np.float64), (n, 3)))
        info = np.zeros(n, dtype=abi.BODY_STEP_INFO_DTYPE)
        contacts = np.zeros((n, max_contacts), dtype=abi.CONTACT_DTYPE)
        _check(self._fn("step_bodies")(self.handle, b.ctypes.data, None if edv is None else edv.ctypes.data, n,
                                       float(dt), g.ctypes.data, info.ctypes.data,
                                       contacts.ctypes.data if max_contacts else None, max_contacts))
        return b, info, contacts

    def step_exposure(self, states, eye_to_world, dt, device: bool = False):
        """exposure::State::step (character/exposure.rs:67-136) against this scene for a batch of eyes: (states,
        exposures).  states: an abi.EXPOSURE_STATE_DTYPE array (see aicb200.exposure_states), stepped by one tick;
        exposures: State::exposure() afterwards, float32 [n].  eye_to_world: [n, 16] float64 (view_transform_matrix per
        eye); dt: Tick::delta_t in seconds, finite and >= 0.  device=True: states is a uint8 CUDA tensor [n, 408] on the
        scene's device (device 0 of a group), stepped in place on its current torch stream, eye_to_world a float64
        tensor [n, 16], and the exposures a float32 tensor."""
        if device:
            torch = _torch()
            dev = self._device()
            n = states.shape[0]
            st = self._tensor(states, torch.uint8, (n, abi.EXPOSURE_STATE_DTYPE.itemsize), "states")
            m = self._tensor(eye_to_world, torch.float64, (n, 16), "eye_to_world")
            out = torch.empty(n, dtype=torch.float32, device=dev)
            _check(self._fn("step_exposure_device")(self.handle, st.data_ptr(), m.data_ptr(), n, float(dt),
                                                     out.data_ptr(), _stream(dev)))
            return st, out
        st = np.ascontiguousarray(states, dtype=abi.EXPOSURE_STATE_DTYPE).copy()
        n = st.shape[0]
        m = np.ascontiguousarray(eye_to_world, dtype=np.float64).reshape(n, 16)
        out = np.zeros(n, dtype=np.float32)
        _check(self._fn("step_exposure")(self.handle, st.ctypes.data, m.ctypes.data, n, float(dt), out.ctypes.data))
        return st, out

    def step_eyes(self, eyes, bodies, dt):
        """step_eye_position (character/eye.rs:90-121) for a batch of eyes after one stepped tick of their bodies, in
        place on the current torch stream.  eyes: a uint8 CUDA tensor [n, 72] of abi.EYE_DTYPE records (see
        aicb200.eyes) on the scene's device (device 0 of a group); bodies: a uint8 tensor [n, 152] of the stepped
        bodies; dt: Tick::delta_t in seconds, in (0, 1].  previous_body_velocity becomes each body's velocity."""
        torch = _torch()
        n = eyes.shape[0]
        e = self._tensor(eyes, torch.uint8, (n, abi.EYE_DTYPE.itemsize), "eyes")
        b = self._tensor(bodies, torch.uint8, (n, abi.BODY_DTYPE.itemsize), "bodies")
        _check(self._fn("step_eyes_device")(self.handle, e.data_ptr(), b.data_ptr(), n, float(dt),
                                             _stream(self._device())))
        return e

    def eye_views(self, eyes, bodies, rotations, exposures, camera_params, eye_to_world=None, cameras=None,
                  look_rays=None, status=None):
        """compute_view_transform (character/eye.rs:187-203) and the world camera's update for a batch of eyes, on the
        current torch stream: each output given is written (None: not written).  eyes and bodies as step_eyes takes
        them; rotations: float64 [n, 4] (look_rotation per eye); exposures: float32 [n] (step_exposure's, device=True)
        or None; camera_params: aicb200.eye_view_params(options, viewport).  Outputs: eye_to_world float64 [n, 16]
        (the next tick's step_exposure input), cameras a uint8 tensor [n, 144] of abi.CAMERA_DTYPE records updated in
        place (see eye_cameras), look_rays float64 [n, 6] (origin, direction at the screen centre) and status int32
        [n] (0, or abi.EYE_NOT_INVERTIBLE).  Returns (eye_to_world, cameras, look_rays, status)."""
        torch = _torch()
        n = eyes.shape[0]
        e = self._tensor(eyes, torch.uint8, (n, abi.EYE_DTYPE.itemsize), "eyes")
        b = self._tensor(bodies, torch.uint8, (n, abi.BODY_DTYPE.itemsize), "bodies")
        r = self._tensor(rotations, torch.float64, (n, 4), "rotations")
        x = None if exposures is None else self._tensor(exposures, torch.float32, (n,), "exposures")
        m = None if eye_to_world is None else self._tensor(eye_to_world, torch.float64, (n, 16), "eye_to_world")
        c = None if cameras is None else self._tensor(cameras, torch.uint8, (n, abi.CAMERA_DTYPE.itemsize), "cameras")
        lr = None if look_rays is None else self._tensor(look_rays, torch.float64, (n, 6), "look_rays")
        st = None if status is None else self._tensor(status, torch.int32, (n,), "status")
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        _check(self._fn("eye_views_device")(self.handle, e.data_ptr(), b.data_ptr(), r.data_ptr(), ptr(x), n,
                                             C.byref(camera_params), ptr(m), ptr(c), ptr(lr), ptr(st),
                                             _stream(self._device())))
        return m, c, lr, st

    def _light_download_device(self):
        torch = _torch()
        dev = self._device()
        out = torch.empty(self.space.size + (4,), dtype=torch.uint8, device=dev)
        _check(self._fn("light_download_device")(self.handle, out.data_ptr(), out.numel() // 4, _stream(dev)))
        return out

    def update_cubes(self, cubes: np.ndarray, block_ids: np.ndarray, light: Optional[np.ndarray] = None):
        """SpaceChange::CubeBlock / CubeLight for a list of cubes; the last entry for a cube wins.  CUDA tensors (int32
        [n, 3], uint16 [n], uint8 [n, 4]) on the scene's device are read where they are, after the work queued on its
        current torch stream."""
        if _is_cuda_tensor(cubes):
            c, ids, lt, n = self._cube_list(cubes, block_ids, light)
            _check(self._fn("scene_update_cubes_device")(self.handle, c.data_ptr(), ids.data_ptr(),
                                                         lt.data_ptr() if lt is not None else None, n,
                                                         _stream(self._device())))
            return
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        ids = np.ascontiguousarray(block_ids, dtype=np.uint16)
        lt = None if light is None else np.ascontiguousarray(light, dtype=np.uint8).reshape(-1, 4)
        _check(self._fn("scene_update_cubes")(self.handle, c.ctypes.data, ids.ctypes.data,
                                              lt.ctypes.data if lt is not None else None, c.shape[0]))

    @staticmethod
    def _region(lower, size, block_ids):
        """A box call's arguments: the region, the dense id array of shape `size` or None, and the uniform id."""
        region = abi.Aab()
        region.lower[:] = [int(v) for v in lower]
        region.size[:] = [int(v) for v in size]
        if np.ndim(block_ids) == 0:
            return region, None, int(block_ids)
        ids = np.ascontiguousarray(block_ids, dtype=np.uint16)
        if ids.shape != tuple(region.size):
            raise ValueError(f"block_ids has shape {ids.shape}, the region {tuple(region.size)}")
        return region, ids, 0

    def update_region(self, lower, size, block_ids, light: Optional[np.ndarray] = None):
        """SpaceChange::CubeBlock (and CubeLight) for every cube of the box (lower, size): update_cubes' box form.
        block_ids: one id for every cube, or an array of shape `size`; light: texels of shape size + (4,), or None.
        Either array may be a CUDA tensor on the scene's device (uint16, uint8), then both are."""
        if _is_cuda_tensor(block_ids) or _is_cuda_tensor(light):
            region, ids, uniform = self._region_device(lower, size, block_ids)
            lt = None if light is None else self._tensor(light, _torch().uint8, tuple(region.size) + (4,), "light")
            _check(self._fn("scene_update_region_device")(self.handle, C.byref(region),
                                                          None if ids is None else ids.data_ptr(), uniform,
                                                          None if lt is None else lt.data_ptr(),
                                                          _stream(self._device())))
            return
        region, ids, uniform = self._region(lower, size, block_ids)
        lt = None if light is None else np.ascontiguousarray(light, dtype=np.uint8)
        if lt is not None and lt.shape != tuple(region.size) + (4,):
            raise ValueError(f"light has shape {lt.shape}, the region {tuple(region.size) + (4,)}")
        _check(self._fn("scene_update_region")(self.handle, C.byref(region), None if ids is None else ids.ctypes.data,
                                               uniform, None if lt is None else lt.ctypes.data))

    def _device_blocks(self, blocks):
        """The aicb_block_desc array and flags of a device call, or None for Blocks; ValueError for a mix."""
        on_device = [isinstance(b, DeviceBlock) for b in blocks]
        if not any(on_device):
            return None
        if not all(on_device):
            raise ValueError("one call takes Blocks or DeviceBlocks, not both")
        device = self._device()
        derive = [b.light is None for b in blocks]
        if any(derive) and not all(derive):
            raise ValueError("one call derives the light of every DeviceBlock (light=None) or of none")
        arr = (abi.BlockDesc * len(blocks))()
        for i, b in enumerate(blocks):
            b._check(device)
            b.fill_desc(arr[i])
        return arr, abi.BLOCKS_DERIVE_LIGHT if derive[0] else 0

    def update_blocks(self, indices, blocks):
        """SpaceChange::BlockEvaluation / BlockIndex: new definitions for existing block indices.  Light is not touched:
        light_relight_blocks(indices) follows it on a lit scene.  DeviceBlocks are read on the device, after the work
        queued on the scene device's current torch stream."""
        idx = np.ascontiguousarray(indices, dtype=np.uint16)
        dev = self._device_blocks(blocks)
        if dev is not None:
            _check(self._fn("scene_update_blocks_device")(self.handle, idx.ctypes.data, dev[0], len(blocks), dev[1],
                                                          _stream(self._device())))
            return
        arr = _block_descs(blocks)
        _check(self._fn("scene_update_blocks")(self.handle, idx.ctypes.data, arr, len(blocks)))

    def append_blocks(self, blocks):
        """SpaceChange::BlockIndex for new indices (UpdatingSpaceRaytracer::update, updating.rs:145-151): the blocks
        become the table's next indices, valid in update_cubes, update_blocks and light_edit_and_propagate.
        DeviceBlocks as in update_blocks."""
        dev = self._device_blocks(blocks)
        if dev is not None:
            _check(self._fn("scene_append_blocks_device")(self.handle, dev[0], len(blocks), dev[1],
                                                          _stream(self._device())))
            return
        arr = _block_descs(blocks)
        _check(self._fn("scene_append_blocks")(self.handle, arr, len(blocks)))

    def fill_uniform(self, block):
        """SpaceChange::EveryBlock (Mutation::fill_uniform over the whole Space): the table becomes [block] and every
        cube holds id 0.  Light is not touched: on a lit scene, light_queue_region(bounds, 210) follows.  A DeviceBlock
        is read on the device, as in update_blocks."""
        dev = self._device_blocks([block])
        if dev is not None:
            _check(self._fn("scene_fill_uniform_device")(self.handle, dev[0], dev[1], _stream(self._device())))
            return
        arr = _block_descs([block])
        _check(self._fn("scene_fill_uniform")(self.handle, arr))

    def upload_light(self, light: np.ndarray):
        """The whole light volume replaced; a CUDA tensor (uint8, Z-major texels) on the scene's device is copied on the
        device."""
        if _is_cuda_tensor(light):
            lt = self._tensor(light, _torch().uint8, tuple(light.shape), "light")
            _check(self._fn("scene_upload_light_device")(self.handle, lt.data_ptr(), lt.numel() // 4,
                                                         _stream(self._device())))
            return
        lt = np.ascontiguousarray(light, dtype=np.uint8).reshape(-1, 4)
        _check(self._fn("scene_upload_light")(self.handle, lt.ctypes.data, lt.shape[0]))

    def set_physics(self, sky_colors, light_max_distance: int):
        """SpaceChange::Physics (Space::set_physics): a new sky (Space's sky_colors: 1 row Uniform, 8 rows Octants) and
        LightPhysics (0 = None, d = Rays { maximum_distance: d }).  A new sky alone leaves the light as it is; a new
        distance reinitialises it (fast_evaluate_light, every cube changed); None frees it."""
        _check(self._fn("scene_set_physics")(self.handle, C.byref(_sky(sky_colors)), light_max_distance))

    # ---- light propagation (space::light; SURVEY 8(a) L1-L4) ----
    def light_fast_evaluate(self):
        """LightStorage::fast_evaluate_light (updater.rs:537-582)"""
        _check(self._fn("light_fast_evaluate")(self.handle))

    def light_compute(self, cubes: np.ndarray) -> np.ndarray:
        """LightStorage::compute_light (updater.rs:368-418) for explicit cubes; returns texels [n,4] in input order."""
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        out = np.zeros((c.shape[0], 4), dtype=np.uint8)
        _check(self._fn("light_compute")(self.handle, c.ctypes.data, c.shape[0], out.ctypes.data))
        return out

    def light_compute_debug(self, cubes: np.ndarray):
        """Space::compute_light::<LightUpdateCubeInfo> (space.rs:810, space/light/debug.rs) for explicit cubes ->
        (texels [n,4] uint8, rays): light_compute's texels, and per cube an array of LIGHT_RAY_DTYPE (LightUpdateRayInfo:
        trigger_cube, value_cube, value, light_from_struck_face) holding the rays that ended on a face opaque for light, in
        the reference's order.  Nothing is stored."""
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        n = c.shape[0]
        texels = np.zeros((n, 4), dtype=np.uint8)
        counts = np.zeros(n, dtype=np.uint32)
        rays = np.zeros(0, dtype=LIGHT_RAY_DTYPE)
        total = C.c_size_t(0)
        fn = self._fn("light_compute_debug")
        status = fn(self.handle, c.ctypes.data, n, texels.ctypes.data, None, 0, counts.ctypes.data, C.byref(total))
        if status == abi.ERR_INVALID and total.value > 0:   # the first call sized the rays
            rays = np.zeros(total.value, dtype=LIGHT_RAY_DTYPE)
            status = fn(self.handle, c.ctypes.data, n, texels.ctypes.data, rays.ctypes.data, rays.size,
                        counts.ctypes.data, C.byref(total))
        _check(status)
        return texels, np.split(rays, np.cumsum(counts.astype(np.int64))[:-1]) if n else []

    def light_evaluate(self, epsilon: int = 0):
        """Mutation::evaluate_light (space.rs:1496-1527) -> (updates, max_difference, chart_node_visits)"""
        n, md, nv = C.c_uint64(0), C.c_uint8(0), C.c_uint64(0)
        _check(self._fn("light_evaluate")(self.handle, epsilon, C.byref(n), C.byref(md), C.byref(nv)))
        return int(n.value), int(md.value), int(nv.value)

    def light_update_from_queue(self, max_updates=None) -> dict:
        """LightStorage::update_light_from_queue (updater.rs:180-290): relaxation rounds until `max_updates` cube updates
        are made or the queue is empty (None: no budget).  Every queued priority >= 1 is eligible; a round that does not
        fit takes the highest priorities first, then the lowest indices.  Returns LightUpdatesInfo (updater.rs:970-984):
        update_count, max_update_difference, queue_count, max_queue_priority."""
        info = abi.LightUpdatesInfo()
        budget = 2**64 - 1 if max_updates is None else int(max_updates)
        _check(self._fn("light_update_from_queue")(self.handle, budget, C.byref(info)))
        return {"update_count": int(info.update_count), "max_update_difference": int(info.max_update_difference),
                "queue_count": int(info.queue_count), "max_queue_priority": int(info.max_queue_priority)}

    def light_edit_cubes(self, cubes: np.ndarray, block_ids: np.ndarray) -> int:
        """Mutation::set(cubes[i], block_ids[i]) in list order, without propagation (light_evaluate or
        light_update_from_queue follows).  A cube may be named more than once.  Returns the number of entries whose id
        differs from the block their cube holds at that point of the list.  CUDA tensors (int32 [n, 3], uint16 [n]) on
        the scene's device are checked and staged on the device."""
        if _is_cuda_tensor(cubes):
            c, ids, _, n = self._cube_list(cubes, block_ids)
            m = C.c_size_t(0)
            _check(self._fn("light_edit_cubes_device")(self.handle, c.data_ptr(), ids.data_ptr(), n, C.byref(m),
                                                       _stream(self._device())))
            return int(m.value)
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        ids = np.ascontiguousarray(block_ids, dtype=np.uint16).reshape(-1)
        if ids.shape[0] != c.shape[0]:
            raise ValueError(f"{c.shape[0]} cubes but {ids.shape[0]} block ids")
        n = C.c_size_t(0)
        _check(self._fn("light_edit_cubes")(self.handle, c.ctypes.data, ids.ctypes.data, c.shape[0], C.byref(n)))
        return int(n.value)

    def light_edit_and_propagate(self, cubes: np.ndarray, block_ids: np.ndarray, epsilon: int = 0):
        """Mutation::set x n + evaluate_light(epsilon) -> (updates, max_difference)"""
        c = np.ascontiguousarray(cubes, dtype=np.int32).reshape(-1, 3)
        ids = np.ascontiguousarray(block_ids, dtype=np.uint16)
        n, md = C.c_uint64(0), C.c_uint8(0)
        _check(self._fn("light_edit_and_propagate")(self.handle, c.ctypes.data, ids.ctypes.data, c.shape[0], epsilon,
                                                    C.byref(n), C.byref(md)))
        return int(n.value), int(md.value)

    def light_edit_region(self, lower, size, block_ids) -> int:
        """Mutation::fill / fill_uniform over the box (lower, size): Mutation::set for every cube, without propagation
        (light_evaluate follows).  block_ids: one id, or an array of shape `size` (a cube the fill leaves alone gets the
        id it holds; a CUDA uint16 tensor on the scene's device is read there).  Returns the number of cubes whose block
        changed."""
        if _is_cuda_tensor(block_ids):
            region, ids, uniform = self._region_device(lower, size, block_ids)
            n = C.c_size_t(0)
            _check(self._fn("light_edit_region_device")(self.handle, C.byref(region), ids.data_ptr(), uniform, C.byref(n),
                                                        _stream(self._device())))
            return int(n.value)
        region, ids, uniform = self._region(lower, size, block_ids)
        n = C.c_size_t(0)
        _check(self._fn("light_edit_region")(self.handle, C.byref(region), None if ids is None else ids.ctypes.data,
                                             uniform, C.byref(n)))
        return int(n.value)

    def light_relight_blocks(self, indices, epsilon: int = 0):
        """The light side of SpaceChange::BlockEvaluation: after update_blocks(indices, ...), Mutation::set's light rule
        (modified_cube_needs_update) for every cube holding one of the indices, then evaluate_light(epsilon)
        -> (updates, max_difference)"""
        idx = np.ascontiguousarray(indices, dtype=np.uint16).reshape(-1)
        n, md = C.c_uint64(0), C.c_uint8(0)
        _check(self._fn("light_relight_blocks")(self.handle, idx.ctypes.data, idx.size, epsilon, C.byref(n),
                                                C.byref(md)))
        return int(n.value), int(md.value)

    def light_stats(self) -> dict:
        """Counters of the last propagation: cube updates, chart node visits, rounds, device seconds."""
        out = (C.c_uint64 * 4)()
        _check(self._fn("light_stats")(self.handle, out))
        return {"cube_updates": int(out[0]), "chart_node_visits": int(out[1]), "rounds": int(out[2]),
                "device_seconds": int(out[3]) * 1e-6}

    def light_changes_count(self) -> int:
        """The number of cubes whose light texel the light calls wrote since the set was last taken
        (SpaceChange::CubeLight, space.rs:1079-1083)."""
        n = C.c_size_t(0)
        _check(self._fn("light_changes_count")(self.handle, C.byref(n)))
        return int(n.value)

    def light_take_changes(self, discard: bool = False):
        """Take the set of changed cubes -> (indices uint32[n], texels uint8[n, 4]): Z-major linear indices in increasing
        order and each cube's texel as it is now.  discard=True empties the set without copying (both arrays empty)."""
        indices = np.zeros(0, dtype=np.uint32)
        texels = np.zeros((0, 4), dtype=np.uint8)
        got = C.c_size_t(0)
        take = self._fn("light_take_changes")
        if discard:
            _check(take(self.handle, None, None, 0, C.byref(got)))
            return indices, texels
        n = self.light_changes_count()
        if n:
            indices = np.zeros(n, dtype=np.uint32)
            texels = np.zeros((n, 4), dtype=np.uint8)
            _check(take(self.handle, indices.ctypes.data, texels.ctypes.data, n, C.byref(got)))
        return indices, texels

    def light_queue_uninitialized(self) -> int:
        """The load rule of Space::new_from_builder (space.rs:290-313): every cube whose texel is Uninitialized (status
        byte 0) enters the light update queue at Priority::UNINIT (210), raise-only.  Returns how many such cubes there
        are.  Nothing propagates: light_evaluate follows."""
        n = C.c_size_t(0)
        _check(self._fn("light_queue_uninitialized")(self.handle, C.byref(n)))
        return int(n.value)

    def light_queue_region(self, lower, size, priority: int):
        """LightStorage::light_needs_update_in_region (updater.rs:122-133): every cube of the box (lower, size) within the
        bounds enters the queue at `priority` (1..255), raise-only."""
        region = abi.Aab()
        region.lower[:] = [int(v) for v in lower]
        region.size[:] = [int(v) for v in size]
        _check(self._fn("light_queue_region")(self.handle, C.byref(region), priority))

    def light_download_queue(self) -> np.ndarray:
        """Each cube's queued priority (0 = not queued), uint8 shaped like the volume."""
        out = np.zeros(self.space.size, dtype=np.uint8)
        _check(self._fn("light_download_queue")(self.handle, out.ctypes.data, out.size, None))
        return out



# ------------------------------------------------------------------------------------------------
# batches of views of one scene (aicb_render_views_* / aicb_group_render_views_*)
# ------------------------------------------------------------------------------------------------
def camera_table(cameras) -> np.ndarray:
    """The aicb_camera records of a list of Camera, as an abi.CAMERA_DTYPE array."""
    table = np.zeros(len(cameras), dtype=abi.CAMERA_DTYPE)
    for v, cam in enumerate(cameras):
        table[v:v + 1].view(np.uint8)[:] = np.frombuffer(bytes(cam.data), dtype=np.uint8)
    return table


def _views_spec(kind, v, h, w, want_depth=False, want_hit=False, want_steps=False) -> dict:
    torch = _torch()
    if kind == "srgb8":
        return {"srgb8": ((v, h, w, 4), torch.uint8)}
    if kind == "rgba16f":
        return {"rgba16f": ((v, h, w, 4), torch.float16)}
    if kind == "text":
        return {"text": ((v, h, w), torch.int32)}
    spec = {"colorbuf": ((v, h * w, 4), torch.float32)}
    if want_depth:
        spec["depth"] = ((v, h * w), torch.float64)
    if want_hit:
        spec["hit"] = ((v, h * w, 8), torch.int32)
    if want_steps:
        spec["steps"] = ((v, h * w), torch.uint32)
    return spec


def _draw_views(scene, group, cameras, options, kind, device, out, size, want_depth=False, want_hit=False,
                want_steps=False):
    """One batch of views on a SpaceRaytracer (group None) or on a DeviceGroup's scene.  kind: srgb8, rgba16f,
    colorbuf or text.  Host: numpy arrays; device: the tensors of _views_spec (a DeviceRendering on one context)."""
    lib = load_library()
    prefix = "aicb_group_" if group is not None else "aicb_"
    opt = options.to_abi(True)
    if device:
        torch = _torch()
        dev = group._device() if group is not None else _ctx_device(scene.ctx)
        if _is_cuda_tensor(cameras):
            if size is None:
                raise ValueError("a camera table tensor needs size=(fb_width, fb_height)")
            w, h = size
            v = cameras.shape[0]
            if (cameras.dtype != torch.uint8 or cameras.device != dev or not cameras.is_contiguous()
                    or tuple(cameras.shape) != (v, abi.CAMERA_DTYPE.itemsize)):
                raise ValueError(f"cameras must be a contiguous uint8 tensor [n, {abi.CAMERA_DTYPE.itemsize}] on {dev}")
            table = cameras
        else:
            v = len(cameras)
            w, h = (cameras[0].data.fb_width, cameras[0].data.fb_height) if v else (0, 0) if size is None else size
            table = torch.from_numpy(camera_table(cameras).view(np.uint8).reshape(v, abi.CAMERA_DTYPE.itemsize)).to(dev)
        t = _device_outputs(out, dev, _views_spec(kind, v, h, w, want_depth, want_hit, want_steps))
        o = _outs_abi(v * w * h, t)
        stream = _stream(dev)
        build = (lambda t, info: _colorbuf_result(t, info)) if kind == "colorbuf" else (lambda t, info: t[kind])
        if group is None:
            return DeviceRendering(scene, lambda held=table: lib.aicb_render_views_device(
                scene.handle, held.data_ptr(), v, w, h, C.byref(opt), C.byref(o), stream), lambda info: build(t, info))
        info = abi.RenderInfo()
        _check(lib.aicb_group_render_views_device(scene.handle if scene else None, table.data_ptr(), v, w, h, C.byref(opt), C.byref(o),
                                                  stream, C.byref(info)))
        return build(t, RenderInfo.from_abi(info))
    table = camera_table(cameras)
    v = len(cameras)
    w, h = (int(table["fb_width"][0]), int(table["fb_height"][0])) if v else (0, 0)
    n = v * w * h
    info = abi.RenderInfo()
    fn = getattr(lib, prefix + "render_views_" + kind)
    handle = scene.handle if scene is not None else None
    if kind == "colorbuf":
        cb = np.empty((v, h * w, 4), dtype=np.float32)
        depth = np.empty((v, h * w), dtype=np.float64) if want_depth else None
        hit = np.empty((v, h * w, 8), dtype=np.int32) if want_hit else None
        steps = np.empty((v, h * w), dtype=np.uint32) if want_steps else None
        _check(fn(handle, table.ctypes.data, v, C.byref(opt), cb.ctypes.data, depth.ctypes.data if want_depth else None,
                  hit.ctypes.data if want_hit else None, steps.ctypes.data if want_steps else None, n, C.byref(info)))
        return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "info": RenderInfo.from_abi(info)}
    shape, dtype = {"srgb8": ((v, h, w, 4), np.uint8), "rgba16f": ((v, h, w, 4), np.float16),
                    "text": ((v, h, w), np.int32)}[kind]
    arr = np.empty(shape, dtype=dtype)
    _check(fn(handle, table.ctypes.data, v, C.byref(opt), arr.ctypes.data, n, C.byref(info)))
    return arr


class _Views:
    """draw_views and its siblings: a batch of cameras of one scene, sharing one GraphicsOptions and one framebuffer
    size, drawn as one frame; view v of the result is the single-camera call's output for cameras[v], bit for bit.
    cameras: a list of Camera, or with device=True a uint8 CUDA tensor [n, 144] of aicb_camera records
    (abi.CAMERA_DTYPE, see camera_table) with size=(fb_width, fb_height).  device=True: the outputs are CUDA tensors
    (out=: the caller's own), as for the other device=True calls."""

    def _views(self, cameras, options, kind, device, out, size, **want):
        raise NotImplementedError

    def draw_views(self, cameras, options, device=False, out=None, size=None):
        """draw_rgba of every camera: uint8 [V, H, W, 4]."""
        return self._views(cameras, options, "srgb8", device, out, size)

    def draw_views_rgba16f(self, cameras, options, device=False, out=None, size=None):
        """draw_rgba16f of every camera: float16 [V, H, W, 4]."""
        return self._views(cameras, options, "rgba16f", device, out, size)

    def draw_views_colorbuf(self, cameras, options, want_depth=True, want_hit=True, want_steps=True, device=False,
                            out=None, size=None):
        """draw_colorbuf of every camera: a dict of colorbuf [V, H * W, 4], depth, hit and steps, and the batch's
        info (counters summed over the views)."""
        return self._views(cameras, options, "colorbuf", device, out, size, want_depth=want_depth, want_hit=want_hit,
                           want_steps=want_steps)

    def render_views_text(self, cameras, options, device=False, out=None, size=None):
        """render_text of every camera: int32 [V, H, W]."""
        return self._views(cameras, options, "text", device, out, size)


class SpaceRaytracer(_Scene, _Views):
    """SpaceRaytracer<()> (sr.rs:51): device-resident snapshot of a Space + graphics options."""

    def __init__(self, space: Space, graphics_options: GraphicsOptions, ctx: Optional[Context] = None):
        self.ctx = ctx or Context.default()
        self.graphics_options = graphics_options.repair()
        self.space = space
        self.handle = C.c_void_p()
        _create_scene("aicb_scene_create", self.ctx.handle, space, _ctx_device(self.ctx), self.handle)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_bytes(self) -> int:
        return int(load_library().aicb_scene_device_bytes(self.handle))

    def trace_rays(self, origin_dir, include_sky: bool = True, want_depth=False, want_hit=False, want_steps=False,
                   out=None):
        """SpaceRaytracer::trace_ray (sr.rs:113-120) over a batch: returns dict of arrays.  With origin_dir a CUDA tensor
        [n, 6] of float64 on the scene's device, the batch is read where it is and the call returns a DeviceRendering
        whose result() is the same dict of tensors (out=: a dict of the caller's own)."""
        if _is_cuda_tensor(origin_dir):
            return _trace_rays_device(self, origin_dir, self.graphics_options.to_abi(include_sky), want_depth, want_hit,
                                      want_steps, out, _ctx_device(self.ctx), None)
        return _trace_rays(self, origin_dir, self.graphics_options.to_abi(include_sky), want_depth, want_hit, want_steps)

    def _device(self):
        return _ctx_device(self.ctx)

    def _views(self, cameras, options, kind, device, out, size, **want):
        self.ctx.settle()
        return _draw_views(self, None, cameras, options, kind, device, out, size, **want)

    def light_download(self, device: bool = False):
        """The light volume, shaped like the Space + (4,): numpy, or with device=True a uint8 tensor on the scene's
        device, ordered before the work queued afterwards on its current torch stream."""
        if device:
            return self._light_download_device()
        out = np.zeros(self.space.size + (4,), dtype=np.uint8)
        _check(load_library().aicb_light_download(self.handle, out.ctypes.data, out.size // 4))
        return out


def _trace_rays(scene, origin_dir, opt, want_depth, want_hit, want_steps) -> dict:
    """aicb_trace_rays on a SpaceRaytracer, aicb_group_trace_rays on a GroupScene."""
    od = np.ascontiguousarray(origin_dir, dtype=np.float64).reshape(-1, 6)
    n = od.shape[0]
    cb = np.empty((n, 4), dtype=np.float32)
    depth = np.empty(n, dtype=np.float64) if want_depth else None
    hit = np.empty((n, 8), dtype=np.int32) if want_hit else None
    steps = np.empty(n, dtype=np.uint32) if want_steps else None
    info = abi.RenderInfo()
    _check(scene._fn("trace_rays")(scene.handle, od.ctypes.data, n, C.byref(opt), cb.ctypes.data,
                                   depth.ctypes.data if want_depth else None, hit.ctypes.data if want_hit else None,
                                   steps.ctypes.data if want_steps else None, C.byref(info)))
    return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "info": RenderInfo.from_abi(info)}


def _is_cuda_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and getattr(x, "is_cuda", False)


def _trace_rays_device(scene, origin_dir, opt, want_depth, want_hit, want_steps, out, device, group):
    """aicb_trace_rays_device on a SpaceRaytracer (a DeviceRendering), aicb_group_trace_rays_device on a group's scene
    (`group`: the dict of tensors)."""
    torch = _torch()
    od = origin_dir.reshape(-1, 6)
    if od.dtype != torch.float64 or od.device != device or not od.is_contiguous():
        raise ValueError(f"origin_dir must be a contiguous float64 tensor [n, 6] on {device}")
    n = od.shape[0]
    t = _device_outputs(out, device, _colorbuf_spec(n, want_depth, want_hit, want_steps))
    o = _outs_abi(n, t)
    lib = load_library()
    stream = _stream(device)
    if group is None:
        return DeviceRendering(scene, lambda: lib.aicb_trace_rays_device(scene.handle, od.data_ptr(), n, C.byref(opt),
                                                                         C.byref(o), stream),
                               lambda info: _colorbuf_result(t, info))
    info = abi.RenderInfo()
    _check(lib.aicb_group_trace_rays_device(scene.handle, od.data_ptr(), n, C.byref(opt), C.byref(o), stream,
                                            C.byref(info)))
    return _colorbuf_result(t, RenderInfo.from_abi(info))


def _layers_device(group, world, ui, backdrop, no_world, spec, out, n, build, depth_transform=None, pixels=None):
    """aicb_render_layers_device (a DeviceRendering) or, with `group` (a DeviceGroup), aicb_group_render_layers_device
    (the result): the outputs of `spec`, n pixels or listed pixels."""
    torch = _torch()
    lead = world if world else ui
    device = torch.device("cuda", group.device_ids[0]) if group is not None else _ctx_device(lead[0].ctx)
    t = _device_outputs(out, device, spec)
    o = _outs_abi(n, t)
    keep = []
    cls = abi.GroupLayer if group is not None else abi.Layer
    w_arg, u_arg = _layer_arg(world, keep, cls), _layer_arg(ui, keep, cls)
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    m = np.ascontiguousarray(depth_transform, dtype=np.float64).reshape(16) if depth_transform is not None else None
    plist = None
    if pixels is not None:   # u32 indices: an int32 or uint32 tensor as it is, anything else converted
        if not _is_cuda_tensor(pixels):   # a list on the host is checked as the host call checks it
            host_px = np.asarray(pixels, dtype=np.int64)
            cam = lead[1].data
            if host_px.size and (host_px.min() < 0 or host_px.max() >= cam.fb_width * cam.fb_height):
                raise AicbError(abi.ERR_INVALID, "pixel index >= fb_width * fb_height")
        plist = pixels if _is_cuda_tensor(pixels) else torch.as_tensor(host_px)
        if plist.dtype not in (torch.int32, torch.uint32):
            plist = plist.to(dtype=torch.int32)
        plist = plist.reshape(-1).to(device=device).contiguous()
    args = (w_arg, u_arg, b.ctypes.data if b is not None else None, nw.ctypes.data if nw is not None else None,
            m.ctypes.data if m is not None else None, plist.data_ptr() if plist is not None else None,
            n if m is not None else 0, C.byref(o))   # the texture's pixels (listed or every one); 0 for frames
    lib = load_library()
    stream = _stream(device)
    if group is None:
        def issue(held=(keep, plist, b, nw, m)):   # what `args` points to stays alive for a re-issue
            return lib.aicb_render_layers_device(*args, stream)
        return DeviceRendering(lead[0], issue, lambda info: build(t, info))
    info = abi.RenderInfo()
    _check(lib.aicb_group_render_layers_device(*args, stream, C.byref(info)))
    return build(t, RenderInfo.from_abi(info))


def _project_cursor(fn, cls, world, ui, ndc, world_max_distance):
    keep = []

    def layer(l):
        if not l:
            return None
        if hasattr(l[0], "ctx"):
            l[0].ctx.settle()
        s = cls(l[0].handle, C.pointer(l[1].data), None)
        keep.append(s)
        return C.byref(s)

    p = np.ascontiguousarray(ndc, dtype=np.float64).reshape(-1, 2)
    out = np.zeros(p.shape[0], dtype=abi.CURSOR_DTYPE)
    _check(fn(layer(world), layer(ui), p.ctypes.data, p.shape[0], float(world_max_distance), out.ctypes.data))
    return out


def project_cursor(world=None, ui=None, ndc=None, world_max_distance: float = 6.0):
    """StandardCameras::project_cursor (stdcam.rs:357-389) for a batch of NDC points [n, 2]: world / ui =
    (SpaceRaytracer, Camera) or None.  Per point the UI layer with f64::INFINITY, then the world layer with
    world_max_distance (the reference hard-codes 6.0); returns an abi.CURSOR_DTYPE array whose `layer` is 1 (UI),
    2 (world) or 0 (nothing)."""
    return _project_cursor(load_library().aicb_project_cursor, abi.Layer, world, ui, ndc, world_max_distance)


NO_WORLD_TO_SHOW_SRGB8 = (0xBC, 0xBC, 0xBC, 0xFF)   # content/palette.rs:76


def _layer_arg(l, keep, cls):
    """(scene, Camera, GraphicsOptions) or None -> a pointer to an aicb_layer / aicb_group_layer (`cls`), kept alive by
    `keep`."""
    if not l:
        return None
    if hasattr(l[0], "ctx"):
        l[0].ctx.settle()
    o = l[2].to_abi(True)
    s = cls(l[0].handle, C.pointer(l[1].data), C.pointer(o))
    keep += [o, s]
    return C.byref(s)


def _layers_srgb8(fn, cls, world, ui, backdrop, no_world) -> "Rendering":
    lead = world if world else ui
    cam = lead[1]
    w, h = cam.data.fb_width, cam.data.fb_height
    keep = []
    out = np.zeros((h, w, 4), dtype=np.uint8)
    info = abi.RenderInfo()
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    _check(fn(_layer_arg(world, keep, cls), _layer_arg(ui, keep, cls), b.ctypes.data if b is not None else None,
              nw.ctypes.data if nw is not None else None, out.ctypes.data, w * h, C.byref(info)))
    return Rendering((w, h), out, int(info.flaws), RenderInfo.from_abi(info))


def render_layers(world=None, ui=None, backdrop=None, no_world=None, device=False, out=None):
    """RtRenderer::draw_rgba through every layer (renderer.rs:282-308, 454-478).
    world / ui = (SpaceRaytracer, Camera, GraphicsOptions) or None; backdrop / no_world = linear RGBA or None.
    device=True: a DeviceRendering whose result() is the Rendering with a uint8 CUDA tensor [H, W, 4] (out=: the
    caller's own)."""
    if device:
        return _layers_srgb8_device(None, world, ui, backdrop, no_world, out)
    return _layers_srgb8(load_library().aicb_render_layers_srgb8, abi.Layer, world, ui, backdrop, no_world)


def _layers_srgb8_device(group, world, ui, backdrop, no_world, out):
    cam = (world if world else ui)[1]
    w, h = cam.data.fb_width, cam.data.fb_height
    return _layers_device(group, world, ui, backdrop, no_world, {"srgb8": ((h, w, 4), _torch().uint8)}, out, w * h,
                          lambda t, info: Rendering((w, h), t["srgb8"], int(info.flaws), info))


def _layers_texture_device(group, world, ui, backdrop, no_world, depth_transform, pixels, out):
    torch = _torch()
    cam = (world if world else ui)[1]
    if pixels is None:
        n = cam.data.fb_width * cam.data.fb_height
    else:
        n = pixels.numel() if _is_cuda_tensor(pixels) else np.asarray(pixels).size
    spec = {"texel_rgba16f": ((n, 4), torch.uint16), "texel_depth": ((n,), torch.float32)}
    return _layers_device(group, world, ui, backdrop, no_world, spec, out, n,
                          lambda t, info: (t["texel_rgba16f"], t["texel_depth"], info), depth_transform, pixels)


def _layers_terminal_device(group, world, ui, backdrop, no_world, out):
    cam = (world if world else ui)[1]
    w, h = cam.data.fb_width, cam.data.fb_height
    return _layers_device(group, world, ui, backdrop, no_world, {"terminal": ((h, w, 6), _torch().int32)}, out, w * h,
                          _terminal_result)


def render_layers_texture(world=None, ui=None, backdrop=None, no_world=None, depth_transform=None, pixels=None,
                          device=False, out=None):
    """RaytraceToTexture::do_some_tracing's trace_one (raytrace_to_texture.rs:591-683) for a batch of pixels, through
    every layer as render_layers traces them.  world / ui = (SpaceRaytracer, Camera, GraphicsOptions) or None;
    depth_transform: [4, 4] (Camera.depth_transform() of the world camera); pixels: linear framebuffer indices
    y * width + x (any order, repeats allowed) or None for the whole texture in row-major order.
    Returns (rgba16f bits uint16 [n, 4], depth float32 [n], RenderInfo); the depth's sign is the pixel's layer (+ world,
    - UI or neither).  device=True: a DeviceRendering whose result() is that triple with CUDA tensors (out=: a dict
    with texel_rgba16f / texel_depth); pixels may then be a CUDA tensor, which is read where it is, unchecked."""
    if device:
        return _layers_texture_device(None, world, ui, backdrop, no_world, depth_transform, pixels, out)
    return _layers_texture(load_library().aicb_render_layers_texture, abi.Layer, world, ui, backdrop, no_world,
                           depth_transform, pixels)


def _layers_texture(fn, cls, world, ui, backdrop, no_world, depth_transform, pixels):
    lead = world if world else ui
    cam = lead[1]
    w, h = cam.data.fb_width, cam.data.fb_height
    keep = []
    m = np.ascontiguousarray(depth_transform, dtype=np.float64).reshape(16)
    if pixels is None:
        n, plist = w * h, None
    else:
        plist = np.ascontiguousarray(pixels, dtype=np.uint32).reshape(-1)
        n = plist.size
    rgba = np.zeros((n, 4), dtype=np.uint16)
    depth = np.zeros(n, dtype=np.float32)
    info = abi.RenderInfo()
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    _check(fn(_layer_arg(world, keep, cls), _layer_arg(ui, keep, cls), b.ctypes.data if b is not None else None,
              nw.ctypes.data if nw is not None else None, m.ctypes.data_as(C.POINTER(C.c_double)),
              plist.ctypes.data if plist is not None else None, n, rgba.ctypes.data, depth.ctypes.data, C.byref(info)))
    return rgba, depth, RenderInfo.from_abi(info)


def render_layers_terminal(world=None, ui=None, backdrop=None, no_world=None, device=False, out=None):
    """The desktop app's terminal frame (all-is-cubes-desktop/src/terminal.rs:114-142): draw::<ColorCharacterBuf>
    through every layer as render_layers traces them, and ColorCharacterBuf::output per pixel.  Same arguments as
    render_layers.  Returns a dict: text (int32 [H, W]: block index, or abi.TEXT_*), layer (int32 [H, W]: the layer
    whose Space a block index belongs to, abi.LAYER_*), rgba (float32 [H, W, 4]: post_process_color(Rgba::from(ColorBuf)),
    linear) and info (RenderInfo).  device=True: a DeviceRendering whose result() is that dict of views of one int32
    CUDA tensor [H, W, 6] (aicb_terminal_pixel; out=: the caller's own)."""
    if device:
        return _layers_terminal_device(None, world, ui, backdrop, no_world, out)
    return _layers_terminal(load_library().aicb_render_layers_terminal, abi.Layer, world, ui, backdrop, no_world)


def _layers_terminal(fn, cls, world, ui, backdrop, no_world) -> dict:
    lead = world if world else ui
    cam = lead[1]
    w, h = cam.data.fb_width, cam.data.fb_height
    keep = []
    out = np.empty((h, w), dtype=[("rgba", np.float32, 4), ("text", np.int32), ("layer", np.int32)])
    assert out.itemsize == C.sizeof(abi.TerminalPixel)
    info = abi.RenderInfo()
    b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
    nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
    _check(fn(_layer_arg(world, keep, cls), _layer_arg(ui, keep, cls), b.ctypes.data if b is not None else None,
              nw.ctypes.data if nw is not None else None, out.ctypes.data, w * h, C.byref(info)))
    # views of the pixels as the call stored them (aicb_terminal_pixel, 24 bytes each)
    return {"text": out["text"], "layer": out["layer"], "rgba": out["rgba"], "info": RenderInfo.from_abi(info)}


CENTRAL_PIXEL_LIMIT = 60000   # raytrace_to_texture.rs:877


def pixel_picker_order(width: int, height: int, count: Optional[int] = None) -> np.ndarray:
    """The pixels RaytraceToTexture's PixelPicker yields (raytrace_to_texture.rs:856-918), as linear indices
    y * width + x: the pixels stably sorted by square radius from the centre plus a 4-level dither, then the first
    min(60000, n / 4) of that order (the centre) cycled interleaved with the rest.  `count` picks (default: one
    cycle_length, after which every pixel has been picked at least once)."""
    n = int(width) * int(height)
    idx = np.arange(n, dtype=np.int64)
    x, y = idx % width, idx // width
    cx, cy = width / 2.0 - 0.5, height / 2.0 - 0.5
    blend = ((x ^ y) % 4 * 2).astype(np.float64)
    square_radius = np.maximum(np.abs(x.astype(np.float64) - cx), np.abs(y.astype(np.float64) - cy))
    key = (square_radius + blend).astype(np.int64)   # `as i64` truncates; the values are >= 0
    sorted_pixels = np.argsort(key, kind="stable")
    central = min(CENTRAL_PIXEL_LIMIT, n // 4)
    inner, outer = central, n - central
    cycle_length = max(inner, outer) * 2
    if count is None:
        count = cycle_length
    if inner == 0 or outer == 0:   # Interleave goes on with the other iterator alone
        length = inner or outer
        lin = (np.arange(count) % length) + (0 if inner else central) if length else np.zeros(0, dtype=np.int64)
    else:
        k = np.arange(count)
        lin = np.where(k % 2 == 0, (k // 2) % inner, central + (k // 2) % outer)
    return sorted_pixels[lin].astype(np.uint32)


def consistent_picks(width: int, height: int, start: int, count: int) -> np.ndarray:
    """The pixels UpdateStrategy::Consistent traces from `next` = start (raytrace_to_texture.rs:704-727): picks
    start .. start + count - 1 through point_from_pixel_index (:912-918), which wraps with rem_euclid / div_euclid, as
    linear indices y * width + x."""
    i = np.uint64(start) + np.arange(count, dtype=np.uint64)
    w, h = np.uint64(width), np.uint64(height)
    return (i % w + (i // w) % h * w).astype(np.uint32)


TEXTURE_INCREMENTAL, TEXTURE_CONSISTENT = abi.TEXTURE_INCREMENTAL, abi.TEXTURE_CONSISTENT


class _DeviceArray:
    """A device buffer the library owns, as __cuda_array_interface__ for torch.as_tensor (no copy); it keeps its owner
    alive as long as a tensor of it lives."""

    def __init__(self, owner, ptr: int, shape, typestr: str):
        self._owner = owner
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False),
                                         "strides": None, "version": 2}


class TextureTarget:
    """RaytraceToTexture's state on the device (raytrace_to_texture.rs): the update strategy and its pick position,
    dirty_pixels, and the colour and depth render targets of RaytraceToTexture::Inner, without the RtRenderer (the
    layers are passed to each trace).  aicb_texture_target_* on a Context, aicb_group_texture_target_* on a DeviceGroup
    (DeviceGroup.texture_target), with the same results.  strategy: TEXTURE_INCREMENTAL (PixelPicker, the reference's)
    or TEXTURE_CONSISTENT (row-major `next`).  rays_per_frame and its time budget stay with the caller, which passes a
    batch size to trace() and times it."""

    def __init__(self, width: int, height: int, strategy: int = TEXTURE_INCREMENTAL, ctx: Optional["Context"] = None,
                 group: Optional["DeviceGroup"] = None):
        self.group = group
        self.ctx = None if group is not None else (ctx or Context.default())
        self._prefix = "aicb_group_texture_target_" if group is not None else "aicb_texture_target_"
        self.handle = C.c_void_p()
        owner = group.handle if group is not None else self.ctx.handle
        _check(self._fn("create")(owner, int(width), int(height), int(strategy), C.byref(self.handle)))

    def _fn(self, name: str):
        if self.ctx is not None:
            self.ctx.settle()
        return getattr(load_library(), self._prefix + name)

    def _device(self):
        return _torch().device("cuda", self.group.device_ids[0] if self.group is not None else self.ctx.device_id)

    def close(self):
        """Destroys the target; a target whose Context was closed first holds nothing that can still be freed."""
        if self.handle and (self.ctx is None or self.ctx.handle):
            self._fn("destroy")(self.handle)
        self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def resize(self, width: int, height: int):
        """UpdateStrategy::resize: the same size does nothing; another makes cleared targets and, for Incremental, a
        new order from pick 0.  dirty_pixels is left as it is."""
        _check(self._fn("resize")(self.handle, int(width), int(height)))

    def mark_dirty(self):
        """RaytraceToTexture::dirty: dirty_pixels = cycle_length."""
        _check(self._fn("mark_dirty")(self.handle))

    def trace(self, world=None, ui=None, backdrop=None, no_world=None, depth_transform=None, n: int = 0):
        """One do_some_tracing batch of n picks: world / ui = (scene, Camera, GraphicsOptions) or None, as
        render_layers_texture takes them (SpaceRaytracers on a Context, GroupScenes on a group).  Returns
        (n_traced, RenderInfo); n_traced is 0 when dirty_pixels was 0, n otherwise."""
        keep = []
        cls = abi.GroupLayer if self.group is not None else abi.Layer
        fn = self._fn("trace")
        w_arg, u_arg = _layer_arg(world, keep, cls), _layer_arg(ui, keep, cls)
        b = np.array(backdrop, dtype=np.float32) if backdrop is not None else None
        nw = np.array(no_world, dtype=np.float32) if no_world is not None else None
        m = np.ascontiguousarray(depth_transform, dtype=np.float64).reshape(16) if depth_transform is not None else None
        traced = C.c_size_t(0)
        info = abi.RenderInfo()
        _check(fn(self.handle, w_arg, u_arg, b.ctypes.data if b is not None else None,
                  nw.ctypes.data if nw is not None else None,
                  m.ctypes.data_as(C.POINTER(C.c_double)) if m is not None else None, int(n), C.byref(traced),
                  C.byref(info)))
        return int(traced.value), RenderInfo.from_abi(info)

    @property
    def state(self) -> dict:
        """width, height, strategy, dirty_pixels, next_pick (the pick position) and cycle_length."""
        s = abi.TextureTargetInfo()
        _check(self._fn("state")(self.handle, C.byref(s)))
        return {"width": s.width, "height": s.height, "strategy": s.strategy, "dirty_pixels": s.dirty_pixels,
                "next_pick": s.next_pick, "cycle_length": s.cycle_length}

    def picks(self, start: int, n: int) -> np.ndarray:
        """The linear pixel indices y * width + x of picks start .. start + n - 1, from the device code that feeds a
        batch."""
        out = np.zeros(int(n), dtype=np.uint32)
        _check(self._fn("picks")(self.handle, int(start), int(n), out.ctypes.data))
        return out

    def read(self):
        """Copies of the targets: (rgba16f bits uint16 [h, w, 4], depth float32 [h, w])."""
        s = self.state
        rgba = np.zeros((s["height"], s["width"], 4), dtype=np.uint16)
        depth = np.zeros((s["height"], s["width"]), dtype=np.float32)
        _check(self._fn("read")(self.handle, rgba.ctypes.data, depth.ctypes.data, s["width"] * s["height"]))
        return rgba, depth

    def tensors(self):
        """The targets in place, as CUDA tensors on the target's device (device 0 of a group): (uint16 [h, w, 4],
        float32 [h, w]).  They stay valid until the next resize() or close(); a later trace() writes into them."""
        torch = _torch()
        s = self.state
        rgba, depth = C.c_void_p(), C.c_void_p()
        _check(self._fn("buffers")(self.handle, C.byref(rgba), C.byref(depth)))
        h, w = s["height"], s["width"]
        dev = self._device()
        return (torch.as_tensor(_DeviceArray(self, rgba.value, (h, w, 4), "<u2"), device=dev),
                torch.as_tensor(_DeviceArray(self, depth.value, (h, w), "<f4"), device=dev))


def render_orthographic(rt, resolution: int = 32) -> "Rendering":
    """raytracer::ortho::render_orthographic (ortho.rs:30-84): the five-view pixel-perfect image of the whole Space.
    `rt`: a SpaceRaytracer, or a GroupScene (its devices share the views' pixels; the same image)."""
    w, h = C.c_uint32(0), C.c_uint32(0)
    _check(rt._fn("ortho_image_size")(rt.handle, resolution, C.byref(w), C.byref(h)))
    out = np.zeros((h.value, w.value, 4), dtype=np.uint8)
    info = abi.RenderInfo()
    _check(rt._fn("render_orthographic")(rt.handle, resolution, out.ctypes.data, w.value * h.value, C.byref(info)))
    return Rendering((w.value, h.value), out, int(info.flaws), RenderInfo.from_abi(info))


def print_space(space: "Space", direction, block_chars: dict, rt=None) -> list:
    """raytracer::print_space (text.rs:139-180): the 80 x 40 character image of a Space seen from `direction`, one
    string per row.  `block_chars` maps a block index to its character (what D::from_block gives each block).
    `rt`: a SpaceRaytracer or a GroupScene of `space` (None: a new SpaceRaytracer)."""
    opts = GraphicsOptions()
    cam = Camera(opts, Viewport((40.0, 40.0), (80, 40)))
    center = [space.lower[a] + space.size[a] / 2.0 for a in range(3)]
    cam.look_at_y_up(eye_for_look_at(space.lower, space.size, direction), center)
    rt = rt or SpaceRaytracer(space, opts)
    o = opts.to_abi(True)
    out = np.zeros(80 * 40, dtype=np.int32)
    _check(rt._fn("render_text")(rt.handle, C.byref(cam.data), C.byref(o), out.ctypes.data, out.size, None))
    special = {abi.TEXT_ENTERED_SPACE: " ", abi.TEXT_EMPTY: ".", abi.TEXT_INCOMPLETE: "X"}
    return ["".join(special[v] if v < 0 else block_chars[int(v)] for v in out[r * 80:(r + 1) * 80]) for r in range(40)]


class GroupScene(_Scene):
    """A Space replicated on every device of a DeviceGroup (aicb_group_scene): what a SpaceRaytracer is to one context,
    kept current by the same updates, applied to every replica, and lit by the same light calls, whose rounds every
    device shares.  Its methods are SpaceRaytracer's, with the same results:

    - Every update and set_physics is validated against replica 0 first: a rejected call changes no replica.
    - light_fast_evaluate, and a set_physics that reinitialises the light, run on device 0; the other replicas take
      copies.  light_compute splits the cubes across the devices.  light_relight_blocks finds the cubes in every
      replica's own cells.
    - The light update queue and the set of changed cubes are device 0's, and the queue calls scan replica 0's volume;
      every replica's texels are identical after every light call.
    - light_stats: the counters of the last light call, summed over the devices; device seconds are device 0's (it
      waits for every device in every round)."""

    _prefix = "aicb_group_"

    def __init__(self, group: "DeviceGroup", space: "Space"):
        self.group = group
        self.space = space
        self.handle = C.c_void_p()
        _create_scene("aicb_group_scene_create", group.handle, space, group._device(), self.handle)

    def _device(self):
        return self.group._device()

    def light_download(self, replica: int = 0, device: bool = False):
        """The light volume of one replica (they are identical after every light call); device=True: replica 0's, as
        a tensor on device 0."""
        if device:
            if replica != 0:
                raise ValueError("device=True downloads replica 0")
            return self._light_download_device()
        out = np.zeros(self.space.size + (4,), dtype=np.uint8)
        _check(load_library().aicb_group_light_download(self.handle, replica, out.ctypes.data, out.size // 4))
        return out


class DeviceGroup(_Views):
    """Several GPUs driven from this one process through the C ABI (csrc/group.cu): scene replicated, frame cut into
    interleaved row strips, pixels stored straight into device 0's frame over NVLink.

    update() / draw(): one world-only scene, which draw_colorbuf() / draw_rgba16f() / trace_rays() / render_text() /
    render_orthographic() also draw, with RtRenderer's and SpaceRaytracer's results.  add_scene() / render_layers() / render_layers_texture() /
    render_layers_terminal(): any number of replicated scenes (GroupScene) drawn through the layers as the module's
    functions of the same names draw them on one context."""

    def __init__(self, device_ids):
        ids = (C.c_int * len(device_ids))(*[int(d) for d in device_ids])
        h = C.c_void_p()
        _check(load_library().aicb_group_create(ids, len(device_ids), C.byref(h)))
        self.handle = h
        self.device_ids = [int(d) for d in device_ids]
        self.scene = None
        self.scenes = []
        self.targets = []

    def add_scene(self, space: "Space") -> GroupScene:
        s = GroupScene(self, space)
        self.scenes.append(s)
        return s

    def _device(self):
        return _torch().device("cuda", self.device_ids[0])

    def project_cursor(self, world=None, ui=None, ndc=None, world_max_distance: float = 6.0):
        """project_cursor with GroupScenes of this group: world / ui = (GroupScene, Camera) or None."""
        return _project_cursor(load_library().aicb_group_project_cursor, abi.GroupLayer, world, ui, ndc,
                               world_max_distance)

    def render_layers(self, world=None, ui=None, backdrop=None, no_world=None, device=False, out=None) -> "Rendering":
        """render_layers with GroupScenes of this group: world / ui = (GroupScene, Camera, GraphicsOptions) or None.
        device=True (here and in the other calls): the outputs are CUDA tensors on device 0 (out=: the caller's own),
        ordered before the work queued afterwards on device 0's current torch stream; the call returns once they are
        final."""
        if device:
            return _layers_srgb8_device(self, world, ui, backdrop, no_world, out)
        return _layers_srgb8(load_library().aicb_group_render_layers_srgb8, abi.GroupLayer, world, ui, backdrop,
                             no_world)

    def render_layers_texture(self, world=None, ui=None, backdrop=None, no_world=None, depth_transform=None,
                              pixels=None, device=False, out=None):
        """render_layers_texture with GroupScenes of this group (same arguments and results)."""
        if device:
            return _layers_texture_device(self, world, ui, backdrop, no_world, depth_transform, pixels, out)
        return _layers_texture(load_library().aicb_group_render_layers_texture, abi.GroupLayer, world, ui, backdrop,
                               no_world, depth_transform, pixels)

    def render_layers_terminal(self, world=None, ui=None, backdrop=None, no_world=None, device=False, out=None) -> dict:
        """render_layers_terminal with GroupScenes of this group (same arguments and results)."""
        if device:
            return _layers_terminal_device(self, world, ui, backdrop, no_world, out)
        return _layers_terminal(load_library().aicb_group_render_layers_terminal, abi.GroupLayer, world, ui, backdrop,
                                no_world)

    def texture_target(self, width: int, height: int, strategy: int = TEXTURE_INCREMENTAL) -> "TextureTarget":
        """A TextureTarget on this group: its targets are device 0's, and a batch is cut across the devices as
        render_layers_texture cuts a pixel list.  Close it before the group."""
        t = TextureTarget(width, height, strategy, group=self)
        self.targets.append(t)
        return t

    def update(self, space: "Space"):
        if self.scene:
            self.scene.close()
            self.scenes.remove(self.scene)
        self.scene = self.add_scene(space)

    def _render_device(self, camera, options, spec, out, build):
        """aicb_group_render_device: the outputs of `spec` for the whole frame, on device 0."""
        device = self._device()
        t = _device_outputs(out, device, spec)
        o = _outs_abi(camera.data.fb_width * camera.data.fb_height, t)
        info = abi.RenderInfo()
        opt = options.to_abi(True)
        _check(load_library().aicb_group_render_device(self._handle(), C.byref(camera.data), C.byref(opt), C.byref(o),
                                                      _stream(device), C.byref(info)))
        return build(t, RenderInfo.from_abi(info))

    def draw(self, camera: "Camera", options: "GraphicsOptions", device=False, out=None) -> "Rendering":
        w, h = camera.data.fb_width, camera.data.fb_height
        if device:
            return self._render_device(camera, options, {"srgb8": ((h, w, 4), _torch().uint8)}, out,
                                       lambda t, info: Rendering((w, h), t["srgb8"], int(info.flaws), info))
        out = np.zeros((h, w, 4), dtype=np.uint8)
        info = abi.RenderInfo()
        o = options.to_abi(True)
        _check(load_library().aicb_group_render_srgb8(self.scene.handle if self.scene else None, C.byref(camera.data),
                                                     C.byref(o), out.ctypes.data, w * h, C.byref(info)))
        return Rendering((w, h), out, int(info.flaws), RenderInfo.from_abi(info))

    def _handle(self):
        return self.scene.handle if self.scene else None

    def _views(self, cameras, options, kind, device, out, size, **want):
        """The batch on the group's scene: view v drawn by device v mod N."""
        return _draw_views(self.scene, self, cameras, options, kind, device, out, size, **want)

    def draw_colorbuf(self, camera: "Camera", options: "GraphicsOptions", want_depth=True, want_hit=True,
                      want_steps=True, device=False, out=None) -> dict:
        """RtRenderer.draw_colorbuf of the whole frame on the group (same dict)."""
        n = camera.data.fb_width * camera.data.fb_height
        if device:
            return self._render_device(camera, options, _colorbuf_spec(n, want_depth, want_hit, want_steps), out,
                                       _colorbuf_result)
        cb = np.empty((n, 4), dtype=np.float32)
        depth = np.empty(n, dtype=np.float64) if want_depth else None
        hit = np.empty((n, 8), dtype=np.int32) if want_hit else None
        steps = np.empty(n, dtype=np.uint32) if want_steps else None
        info = abi.RenderInfo()
        o = options.to_abi(True)
        _check(load_library().aicb_group_render_colorbuf(self._handle(), C.byref(camera.data), C.byref(o),
                                                         cb.ctypes.data, depth.ctypes.data if want_depth else None,
                                                         hit.ctypes.data if want_hit else None,
                                                         steps.ctypes.data if want_steps else None, n, C.byref(info)))
        return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "info": RenderInfo.from_abi(info)}

    def draw_rgba16f(self, camera: "Camera", options: "GraphicsOptions", device=False, out=None) -> np.ndarray:
        """RtRenderer.draw_rgba16f of the whole frame on the group: float16 [h, w, 4]."""
        w, h = camera.data.fb_width, camera.data.fb_height
        if device:
            return self._render_device(camera, options, {"rgba16f": ((h, w, 4), _torch().float16)}, out,
                                       lambda t, info: t["rgba16f"])
        out = np.empty((h, w, 4), dtype=np.float16)
        o = options.to_abi(True)
        _check(load_library().aicb_group_render_rgba16f(self._handle(), C.byref(camera.data), C.byref(o),
                                                        out.ctypes.data, w * h, None))
        return out

    def trace_rays(self, origin_dir, options: "GraphicsOptions", include_sky: bool = True, want_depth=False,
                   want_hit=False, want_steps=False, out=None) -> dict:
        """SpaceRaytracer.trace_rays on the group: the batch is cut into ranges of whole warps, one per device.  A CUDA
        tensor batch on device 0 is read where it is, by every device, and the outputs are tensors on device 0."""
        if not self.scene:
            raise AicbError(abi.ERR_INVALID, "trace_rays() before update()")
        if _is_cuda_tensor(origin_dir):
            return _trace_rays_device(self.scene, origin_dir, options.to_abi(include_sky), want_depth, want_hit,
                                      want_steps, out, self._device(), self)
        return _trace_rays(self.scene, origin_dir, options.to_abi(include_sky), want_depth, want_hit,
                           want_steps)

    def render_text(self, camera: "Camera", options: "GraphicsOptions", device=False, out=None) -> np.ndarray:
        """aicb_group_render_text: per pixel the CharacterBuf state (block index or abi.TEXT_*), int32 [h, w]."""
        w, h = camera.data.fb_width, camera.data.fb_height
        if device:
            return self._render_device(camera, options, {"text": ((h, w), _torch().int32)}, out,
                                       lambda t, info: t["text"])
        out = np.zeros((h, w), dtype=np.int32)
        o = options.to_abi(True)
        _check(load_library().aicb_group_render_text(self._handle(), C.byref(camera.data), C.byref(o), out.ctypes.data,
                                                     w * h, None))
        return out

    def render_orthographic(self, resolution: int = 32) -> "Rendering":
        """render_orthographic of the group's scene."""
        if not self.scene:
            raise AicbError(abi.ERR_INVALID, "render_orthographic() before update()")
        return render_orthographic(self.scene, resolution)

    def close(self):
        for t in self.targets:
            t.close()
        self.targets = []
        for s in self.scenes:
            s.close()
        self.scenes = []
        self.scene = None
        if self.handle:
            load_library().aicb_group_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _shard_abi(shard):
    if shard is None:
        return None
    s = abi.Shard()
    s.strip_rows, s.index, s.count = shard
    return s


class RtRenderer:
    """RtRenderer<()> + impl HeadlessRenderer (renderer.rs:35, 338-355; headless.rs:17-44).

    update(): snapshot the Space onto the GPU (== SpaceRaytracer::new / UpdatingSpaceRaytracer).
    draw(): trace every pixel on the GPU and return a Rendering (== draw_rgba)."""

    def __init__(self, camera: Camera, ctx: Optional[Context] = None):
        self.camera = camera
        self.ctx = ctx or Context.default()
        self.rt: Optional[SpaceRaytracer] = None

    def update(self, space: Space):
        if self.rt is not None:
            self.rt.close()
        self.rt = SpaceRaytracer(space, self.camera.options, self.ctx)

    def _require(self) -> SpaceRaytracer:
        if self.rt is None:
            raise AicbError(abi.ERR_INVALID, "draw() before update()")
        self.rt.ctx.settle()
        return self.rt

    def pixel_count(self, shard=None) -> int:
        s = _shard_abi(shard)
        return int(load_library().aicb_shard_pixel_count(C.byref(self.camera.data), C.byref(s) if s else None))

    def _render_device(self, shard, spec, out, build) -> DeviceRendering:
        """aicb_render_device on the current torch stream: the outputs of `spec` for the shard's pixels."""
        rt = self._require()
        device = _ctx_device(rt.ctx)
        t = _device_outputs(out, device, spec)
        o = _outs_abi(self.pixel_count(shard), t)
        opt = rt.graphics_options.to_abi(True)
        s = _shard_abi(shard)
        stream = _stream(device)
        lib = load_library()
        return DeviceRendering(rt, lambda: lib.aicb_render_device(rt.handle, C.byref(self.camera.data), C.byref(opt),
                                                                  C.byref(s) if s else None, C.byref(o), stream),
                               lambda info: build(t, info))

    def _rows(self, shard):
        n, w = self.pixel_count(shard), self.camera.data.fb_width
        return (n // w if w else 0), w

    def draw(self, info_text: str = "", shard=None, device=False, out=None):
        """draw_rgba.  device=True: a DeviceRendering whose result() is the Rendering with a uint8 CUDA tensor
        [h, w, 4] on the scene's device (out=: the caller's own), issued on the current torch stream; the same holds
        for device=True in draw_rgba16f, draw_colorbuf (out=: a dict) and render_text."""
        if device:
            h, w = self._rows(shard)
            return self._render_device(shard, {"srgb8": ((h, w, 4), _torch().uint8)}, out,
                                       lambda t, info: Rendering((w, h), t["srgb8"], int(info.flaws), info))
        rt = self._require()
        n = self.pixel_count(shard)
        w = self.camera.data.fb_width
        out = np.empty((n, 4), dtype=np.uint8)
        info = abi.RenderInfo()
        opt = rt.graphics_options.to_abi(True)
        s = _shard_abi(shard)
        _check(load_library().aicb_render_srgb8(rt.handle, C.byref(self.camera.data), C.byref(opt),
                                                C.byref(s) if s else None, out.ctypes.data, n, C.byref(info)))
        h = n // w if w else 0
        return Rendering((w, h), out.reshape(h, w, 4) if w else out.reshape(0, 0, 4), int(info.flaws),
                         RenderInfo.from_abi(info))

    draw_rgba = draw

    def draw_rgba16f(self, shard=None, device=False, out=None):
        """The per-pixel colour raytrace_to_texture uploads (raytrace_to_texture.rs:645-661): premultiplied RGBA,
        exposure applied, as float16 [h, w, 4]."""
        if device:
            h, w = self._rows(shard)
            return self._render_device(shard, {"rgba16f": ((h, w, 4), _torch().float16)}, out, lambda t, info: t["rgba16f"])
        rt = self._require()
        n = self.pixel_count(shard)
        w = self.camera.data.fb_width
        out = np.empty((n, 4), dtype=np.float16)
        info = abi.RenderInfo()
        opt = rt.graphics_options.to_abi(True)
        s = _shard_abi(shard)
        _check(load_library().aicb_render_rgba16f(rt.handle, C.byref(self.camera.data), C.byref(opt),
                                                  C.byref(s) if s else None, out.ctypes.data, n, C.byref(info)))
        h = n // w if w else 0
        return out.reshape(h, w, 4) if w else out.reshape(0, 0, 4)

    def draw_colorbuf(self, shard=None, want_depth=True, want_hit=True, want_steps=True, device=False, out=None):
        """RtRenderer::draw::<ColorBuf> (+DepthBuf, +Position) (renderer.rs:183-220)."""
        if device:
            return self._render_device(shard, _colorbuf_spec(self.pixel_count(shard), want_depth, want_hit, want_steps),
                                       out, _colorbuf_result)
        rt = self._require()
        n = self.pixel_count(shard)
        cb = np.empty((n, 4), dtype=np.float32)
        depth = np.empty(n, dtype=np.float64) if want_depth else None
        hit = np.empty((n, 8), dtype=np.int32) if want_hit else None
        steps = np.empty(n, dtype=np.uint32) if want_steps else None
        info = abi.RenderInfo()
        opt = rt.graphics_options.to_abi(True)
        s = _shard_abi(shard)
        _check(load_library().aicb_render_colorbuf(rt.handle, C.byref(self.camera.data), C.byref(opt),
                                                   C.byref(s) if s else None, cb.ctypes.data,
                                                   depth.ctypes.data if want_depth else None,
                                                   hit.ctypes.data if want_hit else None,
                                                   steps.ctypes.data if want_steps else None, n, C.byref(info)))
        return {"colorbuf": cb, "depth": depth, "hit": hit, "steps": steps, "info": RenderInfo.from_abi(info)}

    def render_text(self, device=False, out=None):
        """aicb_render_text of the whole frame: per pixel the CharacterBuf state (block index or abi.TEXT_*), int32
        [h, w]."""
        w, h = self.camera.data.fb_width, self.camera.data.fb_height
        if device:
            return self._render_device(None, {"text": ((h, w), _torch().int32)}, out, lambda t, info: t["text"])
        rt = self._require()
        text = np.zeros((h, w), dtype=np.int32)
        o = rt.graphics_options.to_abi(True)
        _check(load_library().aicb_render_text(rt.handle, C.byref(self.camera.data), C.byref(o), text.ctypes.data, w * h,
                                               None))
        return text


HeadlessRenderer = RtRenderer
