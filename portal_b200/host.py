"""Python handle on the C++ host front-end (include/portal_b200_host.h): scene .ron -> evaluated
uniform table -> scene program -> frames.  Mirrors the reference's `Scene` + `render_frame` call
sequence (/root/reference/src/main.rs:2876-2946); all the work happens in libportal_b200.so."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import PeTarget, PhFrameParams, PortalB200Error, b


class HostScene:
    def __init__(self, ron_text: str):
        self._lib = capi.lib()
        raw = ron_text.encode("utf-8")
        err = C.create_string_buffer(2048)
        self._s = self._lib.ph_scene_load_ron(raw, len(raw), err, len(err))
        if not self._s:
            raise PortalB200Error(err.value.decode(errors="replace"))

    @classmethod
    def from_file(cls, path: str) -> "HostScene":
        with open(path, encoding="utf-8") as f:
            return cls(f.read())

    def close(self):
        if getattr(self, "_s", None):
            self._lib.ph_scene_free(self._s)
            self._s = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise PortalB200Error(self._lib.ph_scene_last_error(self._s).decode(errors="replace"))

    def set_time(self, time: float, total_time: float | None = None):
        self._check(self._lib.ph_scene_set_time(self._s, time, time if total_time is None else total_time))

    def set_value(self, name: str, value: float):
        self._check(self._lib.ph_scene_set_value(self._s, b(name), float(value)))

    def set_formula_camera(self, m16=None):
        """What the `Camera` matrix kind evaluates to; default: the scene's saved camera (what render_frame sends)."""
        if m16 is None:
            cam = self.camera()
            m = (C.c_double * 16)()
            self._lib.ph_orbit_camera_matrix((C.c_double * 3)(*cam["look_at"]), cam["alpha"], cam["beta"], cam["r"], m)
            m16 = list(m)
        self._check(self._lib.ph_scene_set_formula_camera(self._s, (C.c_double * 16)(*m16)))

    def init_stage(self, name: str):
        self._check(self._lib.ph_scene_init_stage(self._s, b(name)))

    def stage_names(self):
        out, nm, k = [], C.c_char_p(), 0
        while self._lib.ph_scene_stage_name(self._s, k, C.byref(nm)) == 0:
            out.append(nm.value.decode())
            k += 1
        return out

    def uniform_table(self) -> dict:
        """name -> ('mat4', [16 f64]) | ('float', f64) | ('int', int), in upload order."""
        n = self._lib.ph_scene_evaluate(self._s)
        if n < 0:
            raise PortalB200Error(self._lib.ph_scene_last_error(self._s).decode(errors="replace"))
        out = {}
        name, typ, vals = C.c_char_p(), C.c_int(), (C.c_double * 16)()
        for k in range(n):
            self._check(self._lib.ph_scene_uniform_get(self._s, k, C.byref(name), C.byref(typ), vals))
            nm = name.value.decode()
            if typ.value == capi.PE_UNIFORM_MAT4:
                out[nm] = ("mat4", [vals[i] for i in range(16)])
            elif typ.value == capi.PE_UNIFORM_FLOAT:
                out[nm] = ("float", vals[0])
            else:
                out[nm] = ("int", int(vals[0]))
        return out

    def camera(self) -> dict:
        la, a, be, r, off = (C.c_double * 3)(), C.c_double(), C.c_double(), C.c_double(), C.c_double()
        self._check(self._lib.ph_scene_camera(self._s, la, C.byref(a), C.byref(be), C.byref(r), C.byref(off)))
        return {"look_at": list(la), "alpha": a.value, "beta": be.value, "r": r.value, "offset_after_material": off.value}

    def textures(self):
        out = []
        name, path = C.c_char_p(), C.c_char_p()
        k = 0
        while self._lib.ph_scene_texture(self._s, k, C.byref(name), C.byref(path)) == 0:
            out.append((name.value.decode(), path.value.decode()))
            k += 1
        return out

    def videos(self):
        """(name, path, uniform name or None) per video: samplers whose image the caller replaces per frame (video.rs:14-20)."""
        out = []
        name, path, uni = C.c_char_p(), C.c_char_p(), C.c_char_p()
        k = 0
        while self._lib.ph_scene_video(self._s, k, C.byref(name), C.byref(path), C.byref(uni)) == 0:
            out.append((name.value.decode(), path.value.decode(), uni.value.decode() or None))
            k += 1
        return out

    def video_frame_index(self, k: int, frame_count: int):
        """VideoRuntime::update (main.rs:862-895): the frame video k shows in the scene's current state, or None."""
        idx = C.c_uint64()
        return int(idx.value) if self._lib.ph_scene_video_frame(self._s, k, frame_count, C.byref(idx)) == 0 else None

    def counts(self) -> dict:
        names = ["objects", "materials", "intersection_materials", "library", "textures", "videos"]
        return {n: self._lib.ph_scene_count(self._s, i) for i, n in enumerate(names)}


class HostPlayer:
    """The animation-facing half of SceneRenderer (ph_player_*, include/portal_b200_host.h): stages, real
    animations, named cameras, time mapping, camera interpolation and -- with a renderer attached -- camera
    teleportation through portals."""

    def __init__(self, scene: HostScene, renderer: "HostRenderer | None" = None):
        self.scene = scene
        self._lib = capi.lib()
        self._p = self._lib.ph_player_new(scene._s)
        if renderer is not None:
            self._check(self._lib.ph_player_attach(self._p, renderer._ctx))
        self.renderer = renderer

    def _check(self, rc):
        if rc != 0:
            raise PortalB200Error(self._lib.ph_player_last_error(self._p).decode(errors="replace"))

    def close(self):
        if getattr(self, "_p", None):
            self._lib.ph_player_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def animations(self):
        """[(name, duration seconds)] in file order."""
        out, nm, d = [], C.c_char_p(), C.c_double()
        for k in range(self._lib.ph_scene_animation_count(self.scene._s)):
            self._lib.ph_scene_animation(self.scene._s, k, C.byref(nm), C.byref(d))
            out.append((nm.value.decode(), d.value))
        return out

    def camera_names(self):
        out, nm = [], C.c_char_p()
        for k in range(self._lib.ph_scene_camera_count(self.scene._s)):
            self._lib.ph_scene_camera_name(self.scene._s, k, C.byref(nm))
            out.append(nm.value.decode())
        return out

    def init_stage(self, name: str):
        self._check(self._lib.ph_player_init_stage(self._p, b(name)))

    def init_animation(self, name: str):
        self._check(self._lib.ph_player_init_animation(self._p, b(name)))

    def select_camera(self, name: str):
        self._check(self._lib.ph_player_select_camera(self._p, b(name)))

    def update(self, time_seconds: float):
        self._check(self._lib.ph_player_update(self._p, float(time_seconds)))

    def set_probe(self, fn):
        """fn(a[3], b[3]) -> (pos[3] | None, encounter_object, change_subspace): teleport_external_ray supplied by the caller
        (tests use the CPU oracle's probe here); None detaches."""
        if fn is None:
            self._check(self._lib.ph_player_set_probe(self._p, None, None))
            self._probe_cb = None
            return

        def tramp(_user, a, b, pos, enc, chg):
            try:
                p, e, c = fn([a[0], a[1], a[2]], [b[0], b[1], b[2]])
                for k in range(3):
                    pos[k] = 0.0 if p is None else float(p[k])
                enc[0], chg[0] = int(bool(e)), int(bool(c))
                return 0
            except Exception:                       # noqa: BLE001 -- must not propagate through the C frame
                return 1

        self._probe_cb = capi.PH_PROBE_FN(tramp)         # keep the trampoline alive
        self._check(self._lib.ph_player_set_probe(self._p, C.cast(self._probe_cb, C.c_void_p), None))

    def set_update_hook(self, fn):
        """fn() after every update the player performs (update() and each motion-blur sub-frame), before the frame's
        uniforms go up: the place to bind the current frame of each video (video_frame_index + pe_set_texture).  An
        exception aborts the call; None detaches."""
        if fn is None:
            self._check(self._lib.ph_player_set_update_hook(self._p, None, None))
            self._hook_cb = None
            return

        def tramp(_user):
            try:
                fn()
                return 0
            except Exception:                       # noqa: BLE001 -- must not propagate through the C frame
                return 1

        self._hook_cb = capi.PH_UPDATE_HOOK(tramp)       # keep the trampoline alive
        self._check(self._lib.ph_player_set_update_hook(self._p, C.cast(self._hook_cb, C.c_void_p), None))

    def set_run_animations(self, on: bool):
        self._check(self._lib.ph_player_set_run_animations(self._p, int(on)))

    def set_stereo(self, draw_side_by_side: bool, eye_distance: float = 0.07, swap_eyes: bool = False):
        self._check(self._lib.ph_player_set_stereo(self._p, int(draw_side_by_side), float(eye_distance), int(swap_eyes)))

    def animation_overrides(self) -> dict:
        """update_inner_variables (main.rs:1696-1755) for the animation entered last: {"render_depth": n | 0, "fps": n | 0}."""
        d, f = C.c_int32(), C.c_int32()
        self._check(self._lib.ph_player_animation_overrides(self._p, C.byref(d), C.byref(f)))
        return {"render_depth": d.value, "fps": f.value}

    def set_anaglyph(self, draw_anaglyph: bool, colorful: bool = False, p: float = 0.29, q: float = 0.06):
        self._check(self._lib.ph_player_set_anaglyph(self._p, int(draw_anaglyph), int(colorful), float(p), float(q)))

    def set_adaptive_aa(self, on: bool, threshold: int = 8):
        """Adaptive anti-aliasing for render_frame and every motion-blur sub-frame (pe_render_adaptive): one sample
        everywhere, all aa_count samples where the one-sample frame's 3x3 unorm8 range exceeds `threshold`."""
        self._check(self._lib.ph_player_set_adaptive_aa(self._p, int(on), int(threshold)))

    def camera_state(self) -> dict:
        cam, inv, orbit, times = (C.c_double * 16)(), (C.c_double * 16)(), (C.c_double * 6)(), (C.c_double * 2)()
        sub, scale, n = C.c_int32(), C.c_double(), C.c_int64()
        self._check(self._lib.ph_player_camera(self._p, cam, inv, C.byref(sub), C.byref(scale), orbit, times, C.byref(n)))
        le, re, ls, rs = (C.c_double * 16)(), (C.c_double * 16)(), C.c_int32(), C.c_int32()
        self._check(self._lib.ph_player_eyes(self._p, le, re, C.byref(ls), C.byref(rs)))
        return {"camera": list(cam), "camera_mul_inv": list(inv), "in_subspace": bool(sub.value), "scale": scale.value,
                "left_eye": list(le), "right_eye": list(re), "left_eye_in_subspace": bool(ls.value),
                "right_eye_in_subspace": bool(rs.value),
                "look_at": list(orbit[:3]), "alpha": orbit[3], "beta": orbit[4], "r": orbit[5],
                "time": times[0], "total_time": times[1], "n_probes": n.value}

    def _render(self, container, bits, width, height, depth, aa_count, aa_start=0, motion_blur=None) -> np.ndarray:
        """ph_player_render: the bytes it writes, as uint8.  motion_blur: (frame_index, frame_count, motion_blur_frames,
        duration_seconds), or None for one frame at the current update."""
        p = PhFrameParams(width, height, depth, aa_count, aa_start, 0)
        mb = None if motion_blur is None else C.byref(capi.PhMotionBlur(*motion_blur))
        cap = self._lib.ph_output_bytes(container, bits, width, height)
        out, n = np.empty(cap, dtype=np.uint8), C.c_size_t()
        self._check(self._lib.ph_player_render(self._p, self.renderer._ctx, C.byref(p), mb, container, bits, out.ctypes.data, cap,
                                               C.byref(n)))
        return out[:n.value]

    def render_frame(self, width, height, depth, aa_count=1, aa_start=0, rgba8=False) -> np.ndarray:
        out = self._render(capi.PH_OUT_PIXELS, 8 if rgba8 else 32, width, height, depth, aa_count, aa_start)
        return out.view(np.uint8 if rgba8 else np.float32).reshape(height, width, 4)

    def render_motion_blur_frame(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                 aa_count=1) -> np.ndarray:
        """One frame of render_animation (main.rs:1786-1817) inside the current animation, RGBA8."""
        mb = (frame_index, frame_count, motion_blur_frames, float(duration_seconds))
        return self._render(capi.PH_OUT_PIXELS, 8, width, height, depth, aa_count, motion_blur=mb).reshape(height, width, 4)

    def advance_motion_blur_frame(self, frame_index, frame_count, motion_blur_frames, duration_seconds):
        """The sub-frame updates of render_motion_blur_frame (same times, order and probes) without the update hook, the
        uniform upload or the render: keeps a player that skips a frame in the state the frame leaves behind."""
        self._check(self._lib.ph_player_advance_motion_blur_frame(self._p, int(frame_index), int(frame_count),
                                                                  int(motion_blur_frames), float(duration_seconds)))

    def render_frame_rgba16(self, width, height, depth, aa_count=1, aa_start=0) -> np.ndarray:
        """The frame of render_frame as unorm16 (uint16 [h, w, 4]): the float frame quantised by pe_quantize_rgba16."""
        return self._render(capi.PH_OUT_PIXELS, 16, width, height, depth, aa_count, aa_start).view(np.uint16).reshape(height, width, 4)

    def render_motion_blur_frame_rgba16(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                        aa_count=1) -> np.ndarray:
        """render_motion_blur_frame with RGBA16 sub-frames and average (uint16 [h, w, 4])."""
        mb = (frame_index, frame_count, motion_blur_frames, float(duration_seconds))
        return self._render(capi.PH_OUT_PIXELS, 16, width, height, depth, aa_count, motion_blur=mb).view(np.uint16).reshape(height, width, 4)

    def render_frame_yuv420p10(self, width, height, depth, bits=8, aa_count=1, aa_start=0):
        """The frame of render_frame (rgba8=True; `bits` 8) or of render_frame_rgba16 (`bits` 16) as Y'CbCr 4:2:0 at 10 bits,
        converted on the device (DESIGN.md section 5.4): (Y, Cb, Cr), numpy uint16 arrays."""
        out = self._render(capi.PH_OUT_YUV420P10, int(bits), width, height, depth, aa_count, aa_start)
        return capi.yuv420p10_planes(out.view(np.uint16), width, height)

    def render_motion_blur_frame_yuv420p10(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                           bits=8, aa_count=1):
        """render_motion_blur_frame (`bits` 8) or render_motion_blur_frame_rgba16 (`bits` 16) as Y'CbCr 4:2:0 planes."""
        mb = (frame_index, frame_count, motion_blur_frames, float(duration_seconds))
        out = self._render(capi.PH_OUT_YUV420P10, int(bits), width, height, depth, aa_count, motion_blur=mb)
        return capi.yuv420p10_planes(out.view(np.uint16), width, height)

    def set_gif_delay(self, delay_cs: int):
        """The Graphic Control Extension delay (centiseconds) of the next GIF frame blocks."""
        self._check(self._lib.ph_player_set_gif_delay(self._p, int(delay_cs)))

    def render_frame_gif(self, width, height, depth, aa_count=1, aa_start=0) -> bytes:
        """The frame of render_frame (rgba8=True) as one GIF frame block encoded on the device (DESIGN.md section 5.6)."""
        return self._render(capi.PH_OUT_GIF, 8, width, height, depth, aa_count, aa_start).tobytes()

    def render_motion_blur_frame_gif(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                     aa_count=1) -> bytes:
        """render_motion_blur_frame as one GIF frame block."""
        mb = (frame_index, frame_count, motion_blur_frames, float(duration_seconds))
        return self._render(capi.PH_OUT_GIF, 8, width, height, depth, aa_count, motion_blur=mb).tobytes()

    def set_apng_frame(self, index: int, delay_num: int, delay_den: int):
        """The frame index and the fcTL delay (delay_num / delay_den seconds) of the next APNG frame blocks."""
        self._check(self._lib.ph_player_set_apng_frame(self._p, int(index), int(delay_num), int(delay_den)))

    def set_jpeg_quality(self, quality: int):
        """The quality (1 .. 100; 90 by default) of the next JPEG frames."""
        self._check(self._lib.ph_player_set_jpeg_quality(self._p, int(quality)))

    def render_frame_jpeg(self, width, height, depth, aa_count=1, aa_start=0) -> bytes:
        """The frame of render_frame (rgba8=True) as a JPEG file encoded on the device (DESIGN.md section 5.7)."""
        return self._render(capi.PH_OUT_JPEG, 8, width, height, depth, aa_count, aa_start).tobytes()

    def render_motion_blur_frame_jpeg(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                      aa_count=1) -> bytes:
        """render_motion_blur_frame as a JPEG file."""
        mb = (frame_index, frame_count, motion_blur_frames, float(duration_seconds))
        return self._render(capi.PH_OUT_JPEG, 8, width, height, depth, aa_count, motion_blur=mb).tobytes()


class HostRenderer:
    """SceneRenderer::new + render_frame over the C API only (no scene IR involved)."""

    def __init__(self, scene: HostScene, device: int = 0, textures: dict | None = None, persistent: bool = False,
                 options: dict | None = None):
        self.scene = scene
        self.device = device
        self._lib = capi.lib()
        self._ctx = self._lib.pe_create(device)
        if not self._ctx:
            raise PortalB200Error("pe_create failed: " + self._lib.pe_last_error(None).decode())
        self._pe(self._lib.pe_set_option(self._ctx, b"persistent", int(persistent)))
        for k, v in (options or {}).items():
            self._pe(self._lib.pe_set_option(self._ctx, b(k), int(v)))
        scene._check(self._lib.ph_scene_build_program(scene._s, self._ctx))
        scene._check(self._lib.ph_scene_upload_uniforms(scene._s, self._ctx))
        for name, arr in (textures or {}).items():
            arr = np.ascontiguousarray(arr, dtype=np.uint8)
            self._pe(self._lib.pe_set_texture(self._ctx, b(name), arr.ctypes.data, arr.shape[1], arr.shape[0]))
        self._pe(self._lib.pe_scene_compile(self._ctx))

    def _pe(self, rc):
        if rc != 0:
            raise PortalB200Error(self._lib.pe_last_error(self._ctx).decode(errors="replace"))

    def source(self) -> str:
        return self._lib.pe_scene_source(self._ctx).decode()

    def render_frame(self, width, height, depth, aa_count=1, aa_start=0, camera=None, rgba8=False) -> np.ndarray:
        p = PhFrameParams(width, height, depth, aa_count, aa_start, 0)
        if camera is not None:
            p.use_camera = 1
            p.look_at = (C.c_double * 3)(*camera["look_at"])
            p.alpha, p.beta, p.r = camera["alpha"], camera["beta"], camera["r"]
        out = np.empty((height, width, 4), dtype=np.uint8 if rgba8 else np.float32)
        self.scene._check(self._lib.ph_render_frame(self.scene._s, self._ctx, C.byref(p), out.ctypes.data, int(rgba8)))
        return out

    def render_target(self, target, out_device_ptr: int, depth: int, aa_count=1, aa_start=0, camera=None, stream: int = 0):
        """ph_render_target: the uniform setup of render_frame, then an asynchronous render of a (row-strip) target into
        device memory (float RGBA); the multi-GPU building block on the host side."""
        p = PhFrameParams(target.width, target.height, depth, aa_count, aa_start, 0)
        if camera is not None:
            p.use_camera = 1
            p.look_at = (C.c_double * 3)(*camera["look_at"])
            p.alpha, p.beta, p.r = camera["alpha"], camera["beta"], camera["r"]
        self.scene._check(self._lib.ph_render_target(self.scene._s, self._ctx, C.byref(p), C.byref(target), out_device_ptr, stream or None))

    def sync(self):
        self._pe(self._lib.pe_sync(self._ctx))

    def frame_uniforms(self, width, height, depth, aa_count=1, aa_start=0, camera=None):
        """ph_frame_uniforms: the per-frame host work of render_frame (float64 scene evaluation + uniform upload) without
        a render; follow with pe_render* / pe_submit_host_rgba8 / a sharder call on self._ctx."""
        p = PhFrameParams(width, height, depth, aa_count, aa_start, 0)
        if camera is not None:
            p.use_camera = 1
            p.look_at = (C.c_double * 3)(*camera["look_at"])
            p.alpha, p.beta, p.r = camera["alpha"], camera["beta"], camera["r"]
        self.scene._check(self._lib.ph_frame_uniforms(self.scene._s, self._ctx, C.byref(p)))

    # the renderer-facing names NativeSharder and the bench use on SceneRenderer exist here too
    def _check(self, rc):
        self._pe(rc)

    def set_uniforms(self):
        pass            # uniforms are uploaded by frame_uniforms()

    def launch_count(self) -> int:
        return int(self._lib.pe_launch_count(self._ctx))

    def render_motion_blur_frame(self, width, height, depth, frame_index, frame_count, motion_blur_frames, duration_seconds,
                                 aa_count=1) -> np.ndarray:
        """One frame of the offline `render` loop (main.rs:1758-1824): sub-frames + gamma-2 average, RGBA8."""
        p = PhFrameParams(width, height, depth, aa_count, 0, 0)
        out = np.empty((height, width, 4), dtype=np.uint8)
        self.scene._check(self._lib.ph_render_motion_blur_frame(self.scene._s, self._ctx, C.byref(p), frame_index, frame_count,
                                                                motion_blur_frames, float(duration_seconds), out.ctypes.data))
        return out

    def set_texture_yuv420(self, name: str, planes, fmt, width: int, height: int):
        """pe_set_texture_yuv420: the Y'CbCr 4:2:0 planes (bytes or a numpy buffer of pe_yuv420_bytes, e.g. one
        Y4MClip.read_frame) converted on the device (DESIGN.md section 5.5) into the image of texture `name`.  `fmt`:
        capi.PeYuvFormat or (bits, matrix, full_range, siting)."""
        f = capi.yuv_format(fmt)
        buf = np.frombuffer(planes, np.uint8) if isinstance(planes, (bytes, bytearray)) else np.ascontiguousarray(planes).view(np.uint8)
        if buf.nbytes < self._lib.pe_yuv420_bytes(width, height, f.bits):
            raise ValueError("the planes are shorter than pe_yuv420_bytes")
        self._pe(self._lib.pe_set_texture_yuv420(self._ctx, b(name), buf.ctypes.data, C.byref(f), width, height))

    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.pe_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Y4MClip:
    """A YUV4MPEG2 clip read one frame at a time (ph_y4m_*, include/portal_b200_host.h): width, height, frame_count, format
    (capi.PeYuvFormat; the matrix is the caller's, "bt709" or "bt601") and partial_bytes (a trailing partial frame, not
    counted)."""

    def __init__(self, path: str, matrix: str = "bt709"):
        self._lib = capi.lib()
        if matrix not in capi.MATRICES:
            raise ValueError("matrix must be bt709 or bt601")
        err = C.create_string_buffer(1024)
        self._r = self._lib.ph_y4m_open(path.encode() if isinstance(path, str) else bytes(path), capi.MATRICES[matrix], err, len(err))
        if not self._r:
            raise PortalB200Error(err.value.decode(errors="replace"))
        w, h, n, part = C.c_int32(), C.c_int32(), C.c_int64(), C.c_int64()
        self.format = capi.PeYuvFormat()
        self._lib.ph_y4m_info(self._r, C.byref(w), C.byref(h), C.byref(n), C.byref(self.format), C.byref(part))
        self.width, self.height, self.frame_count, self.partial_bytes = w.value, h.value, n.value, part.value
        self.frame_bytes = self._lib.pe_yuv420_bytes(self.width, self.height, self.format.bits)

    def read_frame(self, k: int) -> np.ndarray:
        """The planes of frame k as pe_set_texture_yuv420 takes them: a uint8 array of frame_bytes."""
        out = np.empty(self.frame_bytes, np.uint8)
        if self._lib.ph_y4m_read_frame(self._r, int(k), out.ctypes.data, out.nbytes):
            raise PortalB200Error(self._lib.ph_y4m_last_error(self._r).decode(errors="replace"))
        return out

    def planes(self, k: int):
        """(Y [h, w], Cb, Cr [ceil(h/2), ceil(w/2)]) of frame k: uint8 at 8 bits, uint16 at 10."""
        v = self.read_frame(k).view(np.uint8 if self.format.bits == 8 else np.uint16)
        n, cw, ch = self.width * self.height, (self.width + 1) // 2, (self.height + 1) // 2
        return v[:n].reshape(self.height, self.width), v[n:n + cw * ch].reshape(ch, cw), v[n + cw * ch:].reshape(ch, cw)

    def close(self):
        if getattr(self, "_r", None):
            self._lib.ph_y4m_close(self._r)
            self._r = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------ image files either side of the path
def png_decode(data: bytes) -> np.ndarray:
    """PNG file image -> uint8 [h, w, 4] (Texture2D::from_file_with_format, main.rs:1066-1085): ph_png_decode."""
    lib = capi.lib()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data) if data else (C.c_uint8 * 1)()
    out, w, h = C.c_void_p(), C.c_int32(), C.c_int32()
    err = C.create_string_buffer(512)
    if lib.ph_png_decode(buf, len(data), C.byref(out), C.byref(w), C.byref(h), err, len(err)):
        raise PortalB200Error("png: " + err.value.decode(errors="replace"))
    try:
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint8)), shape=(h.value, w.value, 4)).copy()
    finally:
        lib.ph_png_free(out)


def png_encode(rgba8: np.ndarray) -> bytes:
    """uint8 [h, w, 4] -> PNG file image (Image::export_png, main.rs:2939-2943): ph_png_encode_rgba8."""
    lib = capi.lib()
    arr = np.ascontiguousarray(rgba8, dtype=np.uint8)
    if arr.ndim != 3 or arr.shape[2] != 4:
        raise ValueError("frame must be [h, w, 4] uint8")
    out, n = C.c_void_p(), C.c_size_t()
    if lib.ph_png_encode_rgba8(arr.ctypes.data, arr.shape[1], arr.shape[0], C.byref(out), C.byref(n)):
        raise PortalB200Error("png: cannot encode")
    try:
        return C.string_at(out, n.value)
    finally:
        lib.ph_png_free(out)
