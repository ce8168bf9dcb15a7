"""SceneRenderer: host-side mirror of the reference's `SceneRenderer` for the ray-loop path.

Reference interface being mirrored (/root/reference/src/main.rs):
    SceneRenderer::new            :934-1064   build material, set uniforms, set camera, load textures
    SceneRenderer::set_uniforms   :1266-1359  per-frame renderer uniforms (`_camera`, `_ray_tracing_depth`, ...)
    SceneRenderer::draw_texture   :1411-1428  scene.set_uniforms + set_uniforms + draw one rectangle
    render_frame                  :2876-2946  one frame -> RGBA8 image
Field names (aa_count, aa_start, render_depth, offset_after_material, gray_t_start, gray_t_size,
darken_by_distance, angle_color_disable, grid_disable, black_border_disable, draw_depth_map,
depth_map_min/max) are the reference's.

Everything that computes pixels happens in libportal_b200.so (C ABI, include/portal_b200.h) on the
GPU; this module only moves names and numbers across that boundary.  A scene arrives as a
"scene IR" dict: objects / materials / snippets plus the evaluated uniform table (f64), i.e. what
`Scene::set_uniforms` (/root/reference/src/gui/scene.rs:545-658) would upload.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np

from . import capi
from .capi import PeTarget, PortalB200Error, b


def load_scene_ir(path: str) -> dict:
    with open(path) as f:
        return json.load(f)


def load_textures(path: str) -> dict:
    if not os.path.exists(path):
        return {}
    with np.load(path) as z:
        return {k: np.ascontiguousarray(z[k]) for k in z.files}


def orbit_camera_matrix(look_at, alpha, beta, r):
    """RotateAroundCam::get_matrix (/root/reference/src/main.rs:278-304), teleport_matrix = identity,
    free_movement = false.  float64; returns 16 floats, column-major."""
    pv = np.array([math.sin(beta) * math.cos(alpha), math.cos(beta), math.sin(beta) * math.sin(alpha)]) * r
    look_at = np.asarray(look_at, dtype=np.float64)
    pos = pv + look_at

    def norm(v):
        return v * (1.0 / math.sqrt(float(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])))

    k = norm(look_at - pos)
    i = norm(np.cross(k, np.array([0.0, 1.0, 0.0])))
    j = norm(np.cross(k, i))
    m = np.zeros((4, 4))
    m[0, :3], m[1, :3], m[2, :3] = i, j, k
    m[3, :3] = pos
    m[3, 3] = 1.0
    return m.reshape(16)


def camera_scale(cam16) -> float:
    """calc_scale (/root/reference/src/main.rs:1325-1333): mean length of the first three columns."""
    m = np.asarray(cam16, dtype=np.float64).reshape(4, 4)
    return float(sum(math.sqrt(float(np.dot(m[c], m[c]))) for c in range(3)) / 3.0)


class SceneRenderer:
    def __init__(self, scene_ir: dict, textures: dict | None = None, device: int = 0, persistent: bool = False,
                 specialize_ints: bool = True, compile_now: bool = True, options: dict | None = None):
        self.ir = scene_ir
        self.device = device
        self._lib = capi.lib()
        self._ctx = self._lib.pe_create(device)
        if not self._ctx:
            raise PortalB200Error("pe_create failed: " + self._lib.pe_last_error(None).decode())
        # SceneRenderer::new defaults, main.rs:1021-1047
        self.offset_after_material = float(scene_ir["cam"]["offset_after_material"])  # main.rs:1059
        self.gray_t_start = 10.0
        self.gray_t_size = 200.0
        self.render_depth = 100
        self.aa_count = 1
        self.aa_start = 0
        self.draw_depth_map = False
        self.depth_map_min = 0.0
        self.depth_map_max = 10.0
        self.angle_color_disable = False
        self.grid_disable = False
        self.black_border_disable = False
        self.darken_by_distance = True
        self.view_angle = math.pi / 2.0  # RotateAroundCam::new, main.rs:109
        self.camera_in_subspace = False
        self.use_panini_projection = False   # RotateAroundCam::new, main.rs:111-116
        self.panini_param = 1.0
        self.use_360_camera = False
        self.use_180_camera = False
        self.draw_side_by_side = False       # SceneRenderer::new, main.rs:1027
        self.eye_distance = 0.07             # main.rs:1028
        self.draw_anaglyph = False           # main.rs:1030-1033 (the UI toggles them: main.rs:1549-1580)
        self.anaglyph_p = 0.29
        self.anaglyph_q = 0.06
        self.anaglyph_mode = False           # False = grayscale, True = "Colorful anaglyph"
        self.camera_mul_inv = np.eye(4).reshape(16)   # teleport_matrix.inverse(), main.rs:1286-1289
        cam = scene_ir["cam"]
        self.set_cam(cam["look_at"], cam["alpha"], cam["beta"], cam["r"])  # main.rs:1057
        self._check(self._lib.pe_set_option(self._ctx, b"persistent", int(persistent)))
        self._check(self._lib.pe_set_option(self._ctx, b"specialize_ints", int(specialize_ints)))
        for k, v in (options or {}).items():
            self._check(self._lib.pe_set_option(self._ctx, b(k), int(v)))
        self._build_scene()
        self.set_scene_uniforms()
        self.set_uniforms()
        self._tex_keep = []
        for t in scene_ir["textures"]:
            if textures and t["name"] in textures:
                self.set_texture(t["name"], textures[t["name"]])
        if compile_now:
            self.compile()

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc, allow_unknown=False):
        if rc == 0 or (allow_unknown and rc == 2):
            return rc
        raise PortalB200Error(self._lib.pe_last_error(self._ctx).decode(errors="replace"))

    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.pe_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _build_scene(self):
        L, ctx, ir = self._lib, self._ctx, self.ir
        self._check(L.pe_scene_begin(ctx))
        for lib in ir["library"]:
            self._check(L.pe_scene_add_library(ctx, b(lib["name"]), b(lib["code"])))
        d3 = C.c_double * 3
        for m in ir["materials"]:
            t = m["type"]
            if t == "Simple":
                self._check(L.pe_scene_add_material_simple(ctx, b(m["name"]), d3(*m["color"]), m["normal_coef"], int(m["grid"]),
                                                           m["grid_scale"], m["grid_coef"], int(m["grid2"]), int(m["grid3"])))
            elif t == "Reflect":
                self._check(L.pe_scene_add_material_reflect(ctx, b(m["name"]), d3(*m["add_to_color"])))
            elif t == "Refract":
                self._check(L.pe_scene_add_material_refract(ctx, b(m["name"]), d3(*m["add_to_color"]), m["refractive_index"]))
            else:
                self._check(L.pe_scene_add_material_complex(ctx, b(m["name"]), b(m["code"])))
        for o in ir["objects"]:
            if o["class"] == "DebugMatrix":
                self._check(L.pe_scene_add_object_debug_matrix(ctx, b(o["name"]), b(o["matrices"][0])))
                continue
            ma = b(o["matrices"][0])
            mb = b(o["matrices"][1]) if o["kind"] == "Portal" else None
            fn = L.pe_scene_add_object_flat if o["class"] == "Flat" else L.pe_scene_add_object_complex
            self._check(fn(ctx, b(o["name"]), capi.PE_SUBSPACE[o["in_subspace"]], ma, mb, b(o["code"])))
        for im in ir["intersection_materials"]:
            self._check(L.pe_scene_add_intersection_material(ctx, b(im["name"]), b(im["code"])))
        kinds = {"mat4": capi.PE_UNIFORM_MAT4, "float": capi.PE_UNIFORM_FLOAT, "int": capi.PE_UNIFORM_INT}
        for name, u in ir["uniforms"].items():
            self._check(L.pe_scene_declare_uniform(ctx, b(name), kinds[u["type"]]))
        for t in ir["textures"]:
            self._check(L.pe_scene_declare_texture(ctx, b(t["name"])))
        if ir.get("skybox"):
            self._check(L.pe_scene_set_skybox(ctx, b(ir["skybox"])))

    def compile(self):
        self._check(self._lib.pe_scene_compile(self._ctx))

    def source(self) -> str:
        return self._lib.pe_scene_source(self._ctx).decode()

    def cubin(self) -> bytes:
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self._lib.pe_scene_cubin(self._ctx, C.byref(p), C.byref(n)))
        return C.string_at(p, n.value)

    def uniform_block(self, width: int, height: int) -> bytes:
        """Host image of the constant block a width x height render would upload now (uniforms set on this object
        are sent first); the program for it is source()."""
        self.set_uniforms()
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self._lib.pe_scene_uniform_block(self._ctx, width, height, C.byref(p), C.byref(n)))
        return C.string_at(p, n.value)

    def launch_count(self) -> int:
        return int(self._lib.pe_launch_count(self._ctx))

    # ------------------------------------------------------------------ uniforms
    def set_uniform(self, name: str, value):
        """material.set_uniform(name, value): mat4 (16 floats, column-major) | float | int."""
        L, ctx = self._lib, self._ctx
        if isinstance(value, (bool, int, np.integer)):
            return self._check(L.pe_set_uniform_i32(ctx, b(name), int(value)))
        if isinstance(value, (float, np.floating)):
            with np.errstate(over="ignore"):
                return self._check(L.pe_set_uniform_f32(ctx, b(name), float(np.float32(value))))
        with np.errstate(over="ignore", invalid="ignore"):
            arr = np.ascontiguousarray(np.asarray(value, dtype=np.float64).astype(np.float32).reshape(16))
        return self._check(L.pe_set_uniform_mat4(ctx, b(name), arr.ctypes.data_as(C.POINTER(C.c_float))))

    def set_scene_uniforms(self, overrides: dict | None = None):
        """Scene::set_uniforms (scene.rs:545-658): upload the evaluated table (f64 -> f32 / i32)."""
        ov = overrides or {}
        for name, u in self.ir["uniforms"].items():
            v = ov.get(name, u["value"])
            if u["type"] == "int":
                self.set_uniform(name, int(v))
            elif u["type"] == "float":
                self.set_uniform(name, float(v))
            else:
                self.set_uniform(name, v)

    def set_uniform_raw_invalidate(self):
        self._sent_state = None

    def set_cam(self, look_at, alpha, beta, r):
        """RotateAroundCam::set_cam (main.rs:320-332) + get_matrix."""
        self.cam = {"look_at": [float(x) for x in look_at], "alpha": float(alpha), "beta": float(beta), "r": float(r)}
        self.camera_matrix = orbit_camera_matrix(look_at, alpha, beta, r)

    def set_uniforms(self):
        """SceneRenderer::set_uniforms (main.rs:1266-1359), the variants this path implements.
        The reference re-sends all of them every draw; here they are re-sent only when one changed since
        the last call (the library keeps its own copy of the block), which matters once a frame takes
        ~0.1 ms per GPU."""
        state = (tuple(self.camera_matrix), tuple(self.camera_mul_inv), self.camera_in_subspace, self.view_angle, self.render_depth,
                 self.aa_count, self.aa_start, self.draw_depth_map, self.depth_map_min, self.depth_map_max,
                 self.offset_after_material, self.gray_t_start, self.gray_t_size, self.angle_color_disable, self.grid_disable,
                 self.black_border_disable, self.darken_by_distance, self.use_panini_projection, self.panini_param,
                 self.use_360_camera, self.use_180_camera, self.draw_side_by_side, self.eye_distance,
                 self.draw_anaglyph, self.anaglyph_p, self.anaglyph_q, self.anaglyph_mode)
        if state == getattr(self, "_sent_state", None):
            return
        self._sent_state = state
        s = self.set_uniform
        s("_camera", self.camera_matrix)
        s("_camera_in_subspace", int(self.camera_in_subspace))
        s("_view_angle", float(self.view_angle))
        s("_ray_tracing_depth", int(self.render_depth))
        s("_aa_count", int(self.aa_count))
        s("_aa_start", int(self.aa_start))
        s("_draw_depth_map", int(self.draw_depth_map))
        s("_depth_map_min", float(self.depth_map_min))
        s("_depth_map_max", float(self.depth_map_max))
        s("_offset_after_material", float(self.offset_after_material))
        s("_t_start", float(self.gray_t_start))
        s("_t_end", float(self.gray_t_start + self.gray_t_size))
        s("_camera_scale", camera_scale(self.camera_matrix))
        s("_angle_color_disable", int(self.angle_color_disable))
        s("_grid_disable", int(self.grid_disable))
        s("_black_border_disable", int(self.black_border_disable))
        s("_darken_by_distance", int(self.darken_by_distance))
        s("_camera_mul_inv", self.camera_mul_inv)
        s("_use_panini_projection", int(self.use_panini_projection))
        s("_panini_param", float(self.panini_param))
        s("_use_360_camera", int(self.use_360_camera))
        s("_use_180_camera", int(self.use_180_camera))
        s("_draw_side_by_side", int(self.draw_side_by_side))
        s("_draw_anaglyph", int(self.draw_anaglyph))            # main.rs:1308-1315
        s("_anaglyph_p", float(self.anaglyph_p))
        s("_anaglyph_q", float(self.anaglyph_q))
        s("_anaglyph_mode", int(self.anaglyph_mode))
        left, right = self.eye_matrices()
        s("_camera_left_eye", left)
        s("_camera_right_eye", right)
        s("_left_eye_scale", camera_scale(left))
        s("_right_eye_scale", camera_scale(right))
        s("_left_eye_in_subspace", int(self.camera_in_subspace))
        s("_right_eye_in_subspace", int(self.camera_in_subspace))

    def eye_matrices(self):
        """Eye cameras of teleport_eye_matrices (main.rs:1121-1139) when no portal lies between the eyes:
        DMat4::from_translation(C * (+-eye_distance, 0, 0, 1) - cam_pos) * C."""
        c = np.asarray(self.camera_matrix, dtype=np.float64).reshape(4, 4)  # rows = columns of the matrix
        pos = c[3, :3]
        out = []
        for sx in (-1.0, 1.0):
            v = np.array([sx * self.eye_distance, 0.0, 0.0, 1.0])
            p = v @ c                       # C * v with column-major storage
            t = np.eye(4)
            t[3, :3] = p[:3] - pos
            out.append((c @ t).reshape(16))  # T * C in column-major rows
        return out[0], out[1]

    def set_texture(self, name: str, rgba8: np.ndarray):
        arr = np.ascontiguousarray(rgba8, dtype=np.uint8)
        if arr.ndim != 3 or arr.shape[2] != 4:
            raise ValueError("texture must be [h, w, 4] uint8")
        self._check(self._lib.pe_set_texture(self._ctx, b(name), arr.ctypes.data, arr.shape[1], arr.shape[0]))

    # ------------------------------------------------------------------ render
    @staticmethod
    def full_target(width: int, height: int) -> PeTarget:
        return PeTarget(width, height, height, 0, 1, 1, 1)

    @staticmethod
    def strip_target(width: int, height: int, strip_rows: int, rank: int, world: int, full_frame_layout: bool = False) -> PeTarget:
        """Cyclic row strips (SURVEY.md §8e): rank r owns global strips r, r + world, ..."""
        n_global = (height + strip_rows - 1) // strip_rows
        n_local = (n_global - rank + world - 1) // world if rank < n_global else 0
        return PeTarget(width, height, strip_rows, rank, world, max(n_local, 1) if n_local else 0, int(full_frame_layout))

    def draw_texture(self, target: PeTarget, out_ptr: int, bounces_ptr: int = 0, stream: int = 0):
        """draw_texture (main.rs:1411-1428): uniforms + one launch into device memory (async)."""
        self.set_uniforms()
        self._check(self._lib.pe_render(self._ctx, C.byref(target), out_ptr, bounces_ptr or None, stream or None))

    def render_host(self, width: int, height: int, out: np.ndarray | None = None) -> np.ndarray:
        """One frame, float RGBA on the host (the value the reference's shader writes, pre-quantisation)."""
        self.set_uniforms()
        t = self.full_target(width, height)
        if out is None:
            out = np.empty((height, width, 4), dtype=np.float32)
        self._check(self._lib.pe_render_host(self._ctx, C.byref(t), out.ctypes.data))
        return out

    def render_host_ptr(self, width: int, height: int, host_ptr: int, rgba8: bool = True):
        """render_frame's product (main.rs:2929-2943) into caller-owned (pinned) host memory."""
        self.set_uniforms()
        t = self.full_target(width, height)
        fn = self._lib.pe_render_host_rgba8 if rgba8 else self._lib.pe_render_host
        self._check(fn(self._ctx, C.byref(t), host_ptr))

    def draw_texture_rgba8(self, target: PeTarget, out_ptr: int, stream: int = 0):
        """draw_texture into an RGBA8 device buffer: the kernel quantises like the reference's render target."""
        self.set_uniforms()
        self._check(self._lib.pe_render_rgba8(self._ctx, C.byref(target), out_ptr, stream or None))

    def draw_texture_adaptive(self, target: PeTarget, out_ptr: int, threshold: int, rgba8: bool = False, refined_ptr: int = 0,
                              stream: int = 0):
        """Adaptive anti-aliasing into device memory (async, pe_render_adaptive): the one-sample frame, then all aa_count
        samples on the pixels whose 3x3 unorm8 range in it exceeds `threshold`.  `refined_ptr` (optional, device uint32)
        receives the number of refined pixels.  Whole-frame targets only."""
        self.set_uniforms()
        self._check(self._lib.pe_render_adaptive(self._ctx, C.byref(target), int(threshold), int(rgba8), out_ptr, refined_ptr or None,
                                                 stream or None))

    def draw_texture_adaptive_strips(self, target: PeTarget, out_ptr: int, threshold: int, rgba8: bool = False,
                                     refined_ptr: int = 0, stream: int = 0):
        """Adaptive anti-aliasing of any target, strips of a sharded frame included (async, pe_render_adaptive_strips): every
        pixel of the target is the whole-frame adaptive frame's pixel, bit for bit -- the rows next to the strips that other
        ranks own are rendered here at one sample.  `refined_ptr` (optional, device uint32) receives this target's number
        of refined pixels."""
        self.set_uniforms()
        self._check(self._lib.pe_render_adaptive_strips(self._ctx, C.byref(target), int(threshold), int(rgba8), out_ptr,
                                                        refined_ptr or None, stream or None))

    def render_host_adaptive(self, width: int, height: int, threshold: int, rgba8: bool = False) -> tuple[np.ndarray, int]:
        """One adaptive frame on the host (float RGBA, or RGBA8) and the number of refined pixels."""
        n = width * height
        bpp = 4 if rgba8 else 16
        frame = np.empty((height, width, 4), dtype=np.uint8 if rgba8 else np.float32)
        count = np.zeros(1, dtype=np.uint32)
        dev = C.c_void_p()
        self._check(self._lib.pe_device_malloc(self._ctx, n * bpp + 16, C.byref(dev)))
        try:
            cnt_dev = dev.value + n * bpp
            self.draw_texture_adaptive(self.full_target(width, height), dev.value, threshold, rgba8, cnt_dev)
            self._check(self._lib.pe_memcpy_d2h(self._ctx, frame.ctypes.data, dev.value, n * bpp, None))
            self._check(self._lib.pe_memcpy_d2h(self._ctx, count.ctypes.data, cnt_dev, 4, None))
        finally:
            self._lib.pe_device_free(self._ctx, dev)
        return frame, int(count[0])

    def submit_host_rgba8(self, width: int, height: int, host_ptr: int) -> int:
        """Queue one frame (render + D2H into pinned `host_ptr`) and return its ticket; at most
        PE_PIPELINE_DEPTH frames are in flight, frame i's copy overlaps frame i+1's kernel."""
        self.set_uniforms()
        t = self.full_target(width, height)
        ticket = C.c_uint64()
        self._check(self._lib.pe_submit_host_rgba8(self._ctx, C.byref(t), host_ptr, C.byref(ticket)))
        return ticket.value

    def wait_host(self, ticket: int):
        self._check(self._lib.pe_wait_host(self._ctx, ticket))

    def host_malloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.pe_host_malloc(self._ctx, nbytes, C.byref(p)))
        return p.value

    def host_free(self, ptr: int):
        self._check(self._lib.pe_host_free(self._ctx, ptr))

    def render_host_rgba8(self, width: int, height: int) -> np.ndarray:
        out = np.empty((height, width, 4), dtype=np.uint8)
        self.render_host_ptr(width, height, out.ctypes.data, rgba8=True)
        return out

    def probe_ray(self, a, b):
        """teleport_external_ray (main.rs:1361-1409): -> (pos float32[3], have_result, encounter_object, change_subspace)."""
        self.set_uniforms()
        f3 = C.c_float * 3
        pa, pb, out = f3(*[float(np.float32(x)) for x in a]), f3(*[float(np.float32(x)) for x in b]), f3()
        hr, eo, cs = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self._lib.pe_probe_ray(self._ctx, pa, pb, out, C.byref(hr), C.byref(eo), C.byref(cs)))
        return np.array(list(out), dtype=np.float32), bool(hr.value), bool(eo.value), bool(cs.value)

    def sync(self):
        self._check(self._lib.pe_sync(self._ctx))
