"""ctypes binding of the portal_b200 C ABI (include/portal_b200.h).

This is plumbing only: every call goes straight into libportal_b200.so.  There is no Python or
CPU fallback for rendering -- if the library (or a CUDA device) is missing, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libportal_b200.so")

PE_SUBSPACE = {"Normal": 0, "Subspace": 1, "Both": 2}
PE_UNIFORM_MAT4, PE_UNIFORM_FLOAT, PE_UNIFORM_INT = 0, 1, 2


class PeTarget(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("strip_rows", C.c_int32), ("strip_first", C.c_int32),
                ("strip_step", C.c_int32), ("n_strips", C.c_int32), ("full_frame_layout", C.c_int32)]


PH_PROBE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                          C.POINTER(C.c_int32), C.POINTER(C.c_int32))
PH_UPDATE_HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p)


class PhFrameParams(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("depth", C.c_int32), ("aa_count", C.c_int32),
                ("aa_start", C.c_int32), ("use_camera", C.c_int32), ("look_at", C.c_double * 3), ("alpha", C.c_double),
                ("beta", C.c_double), ("r", C.c_double)]


class PhMotionBlur(C.Structure):
    _fields_ = [("frame_index", C.c_int32), ("frame_count", C.c_int32), ("motion_blur_frames", C.c_int32),
                ("duration_seconds", C.c_double)]


PH_OUT_PIXELS, PH_OUT_PNG, PH_OUT_YUV420P10, PH_OUT_GIF, PH_OUT_JPEG, PH_OUT_APNG = 0, 1, 2, 3, 4, 5

PE_YUV_BT709, PE_YUV_BT601 = 0, 1
PE_YUV_SITING_LEFT, PE_YUV_SITING_CENTER = 0, 1
MATRICES = {"bt709": PE_YUV_BT709, "bt601": PE_YUV_BT601}


class PeYuvFormat(C.Structure):
    """pe_yuv_format: bits 8 | 10, matrix PE_YUV_BT709 | PE_YUV_BT601, full_range 0 | 1, siting PE_YUV_SITING_LEFT | CENTER."""
    _fields_ = [("bits", C.c_int), ("matrix", C.c_int), ("full_range", C.c_int), ("siting", C.c_int)]

    def astuple(self):
        return (self.bits, self.matrix, self.full_range, self.siting)


def yuv_format(fmt) -> PeYuvFormat:
    """A PeYuvFormat from itself or from a (bits, matrix, full_range, siting) tuple."""
    return fmt if isinstance(fmt, PeYuvFormat) else PeYuvFormat(*[int(v) for v in fmt])


class PortalB200Error(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load libportal_b200.so (built in-tree by `python -m portal_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PortalB200Error(
            f"{LIB_PATH} is missing: build it with `python -m portal_b200.build` (there is no fallback path)")
    L = C.CDLL(LIB_PATH)
    vp, cp, i32 = C.c_void_p, C.c_char_p, C.c_int
    dbl3 = C.POINTER(C.c_double)
    sig = {
        "pe_create": (vp, [i32]),
        "pe_destroy": (None, [vp]),
        "pe_last_error": (cp, [vp]),
        "pe_abi_version": (i32, []),
        "pe_scene_begin": (i32, [vp]),
        "pe_scene_add_library": (i32, [vp, cp, cp]),
        "pe_scene_add_material_simple": (i32, [vp, cp, dbl3, C.c_double, i32, C.c_double, C.c_double, i32, i32]),
        "pe_scene_add_material_reflect": (i32, [vp, cp, dbl3]),
        "pe_scene_add_material_refract": (i32, [vp, cp, dbl3, C.c_double]),
        "pe_scene_add_material_complex": (i32, [vp, cp, cp]),
        "pe_scene_add_object_flat": (i32, [vp, cp, i32, cp, cp, cp]),
        "pe_scene_add_object_complex": (i32, [vp, cp, i32, cp, cp, cp]),
        "pe_scene_add_object_debug_matrix": (i32, [vp, cp, cp]),
        "pe_scene_add_intersection_material": (i32, [vp, cp, cp]),
        "pe_scene_declare_uniform": (i32, [vp, cp, i32]),
        "pe_scene_declare_texture": (i32, [vp, cp]),
        "pe_scene_set_skybox": (i32, [vp, cp]),
        "pe_scene_compile": (i32, [vp]),
        "pe_scene_source": (cp, [vp]),
        "pe_scene_cubin": (i32, [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]),
        "pe_scene_uniform_block": (i32, [vp, i32, i32, C.POINTER(vp), C.POINTER(C.c_size_t)]),
        "pe_set_option": (i32, [vp, cp, i32]),
        "pe_set_uniform_mat4": (i32, [vp, cp, C.POINTER(C.c_float)]),
        "pe_set_uniform_f32": (i32, [vp, cp, C.c_float]),
        "pe_set_uniform_i32": (i32, [vp, cp, C.c_int32]),
        "pe_set_uniforms_mat4": (i32, [vp, i32, C.POINTER(cp), C.POINTER(C.c_float)]),
        "pe_set_texture": (i32, [vp, cp, vp, i32, i32]),
        "pe_target_pixels": (C.c_size_t, [C.POINTER(PeTarget)]),
        "pe_render": (i32, [vp, C.POINTER(PeTarget), vp, vp, vp]),
        "pe_render_host": (i32, [vp, C.POINTER(PeTarget), vp]),
        "pe_render_host_rgba8": (i32, [vp, C.POINTER(PeTarget), vp]),
        "pe_render_rgba8": (i32, [vp, C.POINTER(PeTarget), vp, vp]),
        "pe_submit_host_rgba8": (i32, [vp, C.POINTER(PeTarget), vp, C.POINTER(C.c_uint64)]),
        "pe_wait_host": (i32, [vp, C.c_uint64]),
        "pe_submit_host_strips_rgba8": (i32, [vp, C.POINTER(PeTarget), vp, C.POINTER(C.c_uint64)]),
        "pe_host_register": (i32, [vp, vp, C.c_size_t]),
        "pe_host_unregister": (i32, [vp, vp]),
        "pe_host_malloc": (i32, [vp, C.c_size_t, C.POINTER(vp)]),
        "pe_host_free": (i32, [vp, vp]),
        "pe_render_adaptive": (i32, [vp, C.POINTER(PeTarget), i32, i32, vp, vp, vp]),
        "pe_render_adaptive_strips": (i32, [vp, C.POINTER(PeTarget), i32, i32, vp, vp, vp]),
        "pe_probe_ray": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32),
                               C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
        "pe_autotune": (i32, [vp, C.POINTER(PeTarget), i32, cp, C.c_size_t]),
        "pe_sync": (i32, [vp]),
        "pe_launch_count": (C.c_uint64, [vp]),
        "pe_deinterleave_strips": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "pe_device_malloc": (i32, [vp, C.c_size_t, C.POINTER(vp)]),
        "pe_device_free": (i32, [vp, vp]),
        "pe_memcpy_d2h": (i32, [vp, vp, vp, C.c_size_t, vp]),
        "pe_scratch_buffer": (i32, [vp, i32, C.c_size_t, C.POINTER(vp)]),
        "pe_signal_u32": (i32, [vp, C.POINTER(vp), i32, C.c_uint32, vp]),
        "pe_stream_wait_geq_u32": (i32, [vp, vp, C.c_uint32, vp]),
        "pe_memset_u32": (i32, [vp, vp, C.c_uint32, C.c_size_t, vp]),
        "pe_ipc_export": (i32, [vp, vp, vp]),
        "pe_ipc_open": (i32, [vp, vp, C.POINTER(vp)]),
        "pe_ipc_close": (i32, [vp, vp]),
        "pe_average_frames_rgba8": (i32, [vp, C.POINTER(vp), i32, vp, C.c_size_t, vp]),
        "pe_quantize_rgba8": (i32, [vp, vp, vp, C.c_size_t, vp]),
        "pe_frames_differ": (i32, [vp, vp, vp, C.c_size_t, vp, C.POINTER(C.c_uint32)]),
        "pe_png_bound": (C.c_size_t, [i32, i32]),
        "pe_encode_png_rgba8": (i32, [vp, vp, i32, i32, vp, C.c_size_t, vp, vp]),
        "pe_encode_png_host": (i32, [vp, vp, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "pe_quantize_rgba16": (i32, [vp, vp, vp, C.c_size_t, vp]),
        "pe_average_frames_rgba16": (i32, [vp, C.POINTER(vp), i32, vp, C.c_size_t, vp]),
        "pe_png_bound_rgba16": (C.c_size_t, [i32, i32]),
        "pe_encode_png_rgba16": (i32, [vp, vp, i32, i32, vp, C.c_size_t, vp, vp]),
        "pe_encode_png_host_rgba16": (i32, [vp, vp, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "pe_gif_frame_bound": (C.c_size_t, [i32, i32]),
        "pe_encode_gif_frame": (i32, [vp, vp, i32, i32, i32, vp, C.c_size_t, vp, vp]),
        "pe_encode_gif_frame_host": (i32, [vp, vp, i32, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "pe_gif_header": (i32, [i32, i32, i32, vp, C.c_size_t]),
        "pe_jpeg_bound": (C.c_size_t, [i32, i32]),
        "pe_apng_frame_bound": (C.c_size_t, [i32, i32, i32]),
        "pe_encode_apng_frame": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, C.c_size_t, vp, vp]),
        "pe_encode_apng_frame_host": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "pe_apng_header": (i32, [i32, i32, i32, C.c_uint32, C.c_uint32, vp, C.c_size_t]),
        "pe_encode_jpeg_rgba8": (i32, [vp, vp, i32, i32, i32, vp, C.c_size_t, vp, vp]),
        "pe_encode_jpeg_host": (i32, [vp, vp, i32, i32, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "pe_yuv420p10_bytes": (C.c_size_t, [i32, i32]),
        "pe_rgba_to_yuv420p10": (i32, [vp, vp, i32, i32, i32, vp, vp]),
        "pe_yuv420_bytes": (C.c_size_t, [i32, i32, i32]),
        "pe_yuv420_to_rgba8": (i32, [vp, vp, C.POINTER(PeYuvFormat), i32, i32, vp, vp]),
        "pe_set_texture_yuv420": (i32, [vp, cp, vp, C.POINTER(PeYuvFormat), i32, i32]),
        "pe_shard_target": (i32, [i32, i32, i32, i32, i32, i32, C.POINTER(PeTarget)]),
        "pe_sharder_create": (i32, [vp, cp, i32, i32, i32, i32, i32, i32, i32, C.POINTER(vp)]),
        "pe_sharder_destroy": (None, [vp]),
        "pe_sharder_last_error": (cp, [vp]),
        "pe_sharder_target": (i32, [vp, C.POINTER(PeTarget)]),
        "pe_sharder_render": (i32, [vp, vp, C.POINTER(vp)]),
        "pe_sharder_release": (i32, [vp, vp]),
        "pe_sharder_render_overlapped": (i32, [vp, vp, C.POINTER(vp)]),
        "pe_sharder_flush": (i32, [vp, vp, C.POINTER(vp)]),
        "pe_sharder_set_adaptive_aa": (i32, [vp, i32, i32]),
        "pe_sharder_submit": (i32, [vp, C.POINTER(C.c_uint64)]),
        "pe_sharder_complete": (i32, [vp, C.c_uint64]),
        "pe_sharder_wait_frame": (i32, [vp, C.c_uint64, C.POINTER(vp)]),
        "pe_sharder_release_frame": (i32, [vp, C.c_uint64]),
    }
    f64p = C.POINTER(C.c_double)
    sig.update({
        "ph_scene_load_ron": (vp, [cp, C.c_size_t, C.c_char_p, C.c_size_t]),
        "ph_scene_free": (None, [vp]),
        "ph_scene_last_error": (cp, [vp]),
        "ph_scene_set_time": (i32, [vp, C.c_double, C.c_double]),
        "ph_scene_set_value": (i32, [vp, cp, C.c_double]),
        "ph_scene_set_formula_camera": (i32, [vp, f64p]),
        "ph_scene_init_stage": (i32, [vp, cp]),
        "ph_scene_stage_name": (i32, [vp, i32, C.POINTER(cp)]),
        "ph_scene_evaluate": (i32, [vp]),
        "ph_scene_uniform_get": (i32, [vp, i32, C.POINTER(cp), C.POINTER(i32), f64p]),
        "ph_scene_camera": (i32, [vp, f64p, f64p, f64p, f64p, f64p]),
        "ph_scene_texture": (i32, [vp, i32, C.POINTER(cp), C.POINTER(cp)]),
        "ph_scene_count": (i32, [vp, i32]),
        "ph_player_set_update_hook": (i32, [vp, vp, vp]),
        "ph_png_decode": (i32, [vp, C.c_size_t, C.POINTER(vp), C.POINTER(i32), C.POINTER(i32), cp, C.c_size_t]),
        "ph_png_encode_rgba8": (i32, [vp, i32, i32, C.POINTER(vp), C.POINTER(C.c_size_t)]),
        "ph_png_free": (None, [vp]),
        "ph_video_frames_dir": (i32, [cp, cp, C.c_size_t]),
        "ph_scene_video": (i32, [vp, i32, C.POINTER(cp), C.POINTER(cp), C.POINTER(cp)]),
        "ph_scene_video_frame": (i32, [vp, i32, C.c_uint64, C.POINTER(C.c_uint64)]),
        "ph_scene_build_program": (i32, [vp, vp]),
        "ph_scene_upload_uniforms": (i32, [vp, vp]),
        "ph_orbit_camera_matrix": (None, [f64p, C.c_double, C.c_double, C.c_double, f64p]),
        "ph_camera_scale": (C.c_double, [f64p]),
        "ph_render_frame": (i32, [vp, vp, C.POINTER(PhFrameParams), vp, i32]),
        "ph_frame_uniforms": (i32, [vp, vp, C.POINTER(PhFrameParams)]),
        "ph_render_target": (i32, [vp, vp, C.POINTER(PhFrameParams), C.POINTER(PeTarget), vp, vp]),
        "ph_render_motion_blur_frame": (i32, [vp, vp, C.POINTER(PhFrameParams), i32, i32, i32, C.c_double, vp]),
        "ph_player_new": (vp, [vp]),
        "ph_player_free": (None, [vp]),
        "ph_player_last_error": (cp, [vp]),
        "ph_player_attach": (i32, [vp, vp]),
        "ph_player_set_probe": (i32, [vp, vp, vp]),
        "ph_player_init_stage": (i32, [vp, cp]),
        "ph_player_init_animation": (i32, [vp, cp]),
        "ph_player_select_camera": (i32, [vp, cp]),
        "ph_player_update": (i32, [vp, C.c_double]),
        "ph_player_camera": (i32, [vp, f64p, f64p, C.POINTER(i32), f64p, f64p, f64p, C.POINTER(C.c_int64)]),
        "ph_player_set_stereo": (i32, [vp, i32, C.c_double, i32]),
        "ph_player_set_run_animations": (i32, [vp, i32]),
        "ph_player_animation_overrides": (i32, [vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
        "ph_player_set_anaglyph": (i32, [vp, i32, i32, C.c_double, C.c_double]),
        "ph_player_eyes": (i32, [vp, f64p, f64p, C.POINTER(i32), C.POINTER(i32)]),
        "ph_scene_animation_count": (i32, [vp]),
        "ph_scene_animation": (i32, [vp, i32, C.POINTER(cp), f64p]),
        "ph_scene_camera_count": (i32, [vp]),
        "ph_scene_camera_name": (i32, [vp, i32, C.POINTER(cp)]),
        "ph_output_bytes": (C.c_size_t, [i32, i32, i32, i32]),
        "ph_player_render": (i32, [vp, vp, C.POINTER(PhFrameParams), C.POINTER(PhMotionBlur), i32, i32, vp, C.c_size_t,
                                   C.POINTER(C.c_size_t)]),
        "ph_player_advance_motion_blur_frame": (i32, [vp, i32, i32, i32, C.c_double]),
        "ph_player_set_adaptive_aa": (i32, [vp, i32, i32]),
        "ph_player_set_gif_delay": (i32, [vp, i32]),
        "ph_player_set_jpeg_quality": (i32, [vp, i32]),
        "ph_player_set_apng_frame": (i32, [vp, i32, i32, i32]),
        "ph_y4m_open": (vp, [cp, i32, cp, C.c_size_t]),
        "ph_y4m_info": (i32, [vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(PeYuvFormat),
                              C.POINTER(C.c_int64)]),
        "ph_y4m_read_frame": (i32, [vp, C.c_int64, vp, C.c_size_t]),
        "ph_y4m_last_error": (cp, [vp]),
        "ph_y4m_close": (None, [vp]),
    })
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def exported_symbols():
    """Names bound above (tests compare them with include/portal_b200.h)."""
    lib()
    return sorted(n for n in dir(_lib) if n.startswith(("pe_", "ph_")))


def b(s: str) -> bytes:
    return s.encode("utf-8")


def _encode_png(ctx, frame, dtype: str, bound: str, encode: str) -> bytes:
    if frame.dim() != 3 or frame.shape[2] != 4 or not frame.is_cuda or str(frame.dtype) != f"torch.{dtype}" or not frame.is_contiguous():
        raise ValueError(f"frame must be a contiguous CUDA {dtype} tensor [h, w, 4]")
    L = lib()
    h, w = int(frame.shape[0]), int(frame.shape[1])
    cap = getattr(L, bound)(w, h)
    if cap == 0:
        raise PortalB200Error(f"{bound}: no PNG for a {w} x {h} frame")
    out, n = (C.c_uint8 * cap)(), C.c_size_t()
    if getattr(L, encode)(ctx, C.c_void_p(frame.data_ptr()), w, h, out, cap, C.byref(n)):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    return bytes(memoryview(out)[:n.value])


def encode_png_device(ctx, rgba8) -> bytes:
    """PNG file of a CUDA uint8 tensor [h, w, 4] (contiguous) encoded on the device by pe_encode_png_host on context `ctx`
    (a pe_ctx pointer: SceneRenderer._ctx / HostRenderer._ctx)."""
    return _encode_png(ctx, rgba8, "uint8", "pe_png_bound", "pe_encode_png_host")


def encode_png16_device(ctx, rgba16) -> bytes:
    """16-bit PNG file of a CUDA uint16 tensor [h, w, 4] (contiguous, host byte order) encoded on the device by
    pe_encode_png_host_rgba16 on context `ctx`."""
    return _encode_png(ctx, rgba16, "uint16", "pe_png_bound_rgba16", "pe_encode_png_host_rgba16")


def encode_gif_frame(ctx, rgba8, delay_cs: int = 0) -> bytes:
    """GIF frame block (DESIGN.md section 5.6) of a CUDA uint8 tensor [h, w, 4] (contiguous) encoded on the device by
    pe_encode_gif_frame on context `ctx`, ordered after the work already queued on the current torch stream.  A file is
    gif_header(w, h, loop) + the blocks + b"\\x3b"."""
    return _encode_on_stream(ctx, rgba8, "GIF frame", "pe_gif_frame_bound", "pe_encode_gif_frame", int(delay_cs))


def encode_jpeg(ctx, rgba8, quality: int = 90) -> bytes:
    """JPEG file (DESIGN.md section 5.7) of a CUDA uint8 tensor [h, w, 4] (contiguous; alpha ignored) at `quality` 1 .. 100,
    encoded on the device by pe_encode_jpeg_rgba8 on context `ctx`, ordered after the work already queued on the current torch
    stream."""
    return _encode_on_stream(ctx, rgba8, "JPEG", "pe_jpeg_bound", "pe_encode_jpeg_rgba8", int(quality))


def _encode_on_stream(ctx, rgba8, what: str, bound: str, encode: str, arg: int) -> bytes:
    import torch
    if rgba8.dim() != 3 or rgba8.shape[2] != 4 or not rgba8.is_cuda or rgba8.dtype != torch.uint8 or not rgba8.is_contiguous():
        raise ValueError("frame must be a contiguous CUDA uint8 tensor [h, w, 4]")
    L = lib()
    h, w = int(rgba8.shape[0]), int(rgba8.shape[1])
    cap = getattr(L, bound)(w, h)
    if cap == 0:
        raise PortalB200Error(f"{bound}: no {what} for a {w} x {h} frame")
    out = torch.empty(cap, dtype=torch.uint8, device=rgba8.device)
    size = torch.empty(1, dtype=torch.int64, device=rgba8.device)
    # the read-backs go on the same stream handle (0, torch's default stream, names the context's stream)
    stream = C.c_void_p(torch.cuda.current_stream(rgba8.device).cuda_stream)
    n = C.c_uint64()
    if (getattr(L, encode)(ctx, C.c_void_p(rgba8.data_ptr()), w, h, arg, C.c_void_p(out.data_ptr()), cap,
                           C.c_void_p(size.data_ptr()), stream)
            or L.pe_memcpy_d2h(ctx, C.addressof(n), C.c_void_p(size.data_ptr()), 8, stream)):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    host = (C.c_uint8 * max(1, n.value))()
    if L.pe_memcpy_d2h(ctx, host, C.c_void_p(out.data_ptr()), n.value, stream):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    return bytes(host[:n.value])


def encode_apng_frame(ctx, pixels, index: int = 0, delay_num: int = 0, delay_den: int = 1) -> bytes:
    """APNG frame block `index` (DESIGN.md section 5.8) of a CUDA uint8 (8-bit) or uint16 (16-bit, host byte order) tensor
    [h, w, 4] (contiguous) with the delay delay_num / delay_den seconds, encoded on the device by pe_encode_apng_frame on
    context `ctx`, ordered after the work already queued on the current torch stream.  A file is
    apng_header(w, h, bits, n) + blocks 0 .. n - 1 + IEND."""
    import torch
    if (pixels.dim() != 3 or pixels.shape[2] != 4 or not pixels.is_cuda or pixels.dtype not in (torch.uint8, torch.uint16)
            or not pixels.is_contiguous()):
        raise ValueError("frame must be a contiguous CUDA uint8 or uint16 tensor [h, w, 4]")
    L = lib()
    bits = 8 if pixels.dtype == torch.uint8 else 16
    h, w = int(pixels.shape[0]), int(pixels.shape[1])
    cap = L.pe_apng_frame_bound(w, h, bits)
    if cap == 0:
        raise PortalB200Error(f"pe_apng_frame_bound: no APNG frame for a {w} x {h} frame at {bits} bits")
    out = torch.empty(cap, dtype=torch.uint8, device=pixels.device)
    size = torch.empty(1, dtype=torch.int64, device=pixels.device)
    # the read-backs go on the same stream handle (0, torch's default stream, names the context's stream)
    stream = C.c_void_p(torch.cuda.current_stream(pixels.device).cuda_stream)
    n = C.c_uint64()
    if (L.pe_encode_apng_frame(ctx, C.c_void_p(pixels.data_ptr()), w, h, bits, int(index), int(delay_num), int(delay_den),
                               C.c_void_p(out.data_ptr()), cap, C.c_void_p(size.data_ptr()), stream)
            or L.pe_memcpy_d2h(ctx, C.addressof(n), C.c_void_p(size.data_ptr()), 8, stream)):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    host = (C.c_uint8 * max(1, n.value))()
    if L.pe_memcpy_d2h(ctx, host, C.c_void_p(out.data_ptr()), n.value, stream):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    return bytes(host[:n.value])


def apng_header(width: int, height: int, bits: int, num_frames: int, num_plays: int = 0) -> bytes:
    """The APNG file header pe_apng_header writes: the PNG signature, IHDR at `bits` 8 or 16 and acTL."""
    buf = (C.c_uint8 * 64)()
    n = lib().pe_apng_header(width, height, bits, num_frames, num_plays, buf, 64)
    if n == 0:
        raise PortalB200Error(f"pe_apng_header: no APNG header for a {width} x {height} frame at {bits} bits, {num_frames} frames")
    return bytes(buf[:n])


APNG_TRAILER = b"\x00\x00\x00\x00IEND\xaeB`\x82"


def gif_header(width: int, height: int, loop: bool) -> bytes:
    """The GIF file header pe_gif_header writes: GIF89a, the logical screen descriptor and, for an animation, the loop block."""
    buf = (C.c_uint8 * 64)()
    n = lib().pe_gif_header(width, height, 1 if loop else 0, buf, 64)
    if n == 0:
        raise PortalB200Error(f"pe_gif_header: no GIF header for a {width} x {height} frame")
    return bytes(buf[:n])


def yuv420p10_planes(buf, width: int, height: int):
    """Split the planes pe_rgba_to_yuv420p10 writes (a uint16 array of pe_yuv420p10_bytes / 2 values) into Y [h, w],
    Cb and Cr [ceil(h/2), ceil(w/2)]."""
    cw, ch = (width + 1) // 2, (height + 1) // 2
    n = width * height
    return (buf[:n].reshape(height, width), buf[n:n + cw * ch].reshape(ch, cw), buf[n + cw * ch:n + 2 * cw * ch].reshape(ch, cw))


def yuv420p10_device(ctx, rgba, bits: int):
    """Y'CbCr 4:2:0 10-bit planes (DESIGN.md section 5.4) of a CUDA uint8 (`bits` 8) or uint16 (`bits` 16) tensor [h, w, 4]
    (contiguous), converted on the device by pe_rgba_to_yuv420p10 on context `ctx`, ordered after the work already queued on
    the current torch stream.  Returns (Y, Cb, Cr) as numpy uint16 arrays."""
    import numpy as np
    import torch
    want = {8: torch.uint8, 16: torch.uint16}.get(bits)
    if want is None:
        raise ValueError("bits must be 8 or 16")
    if rgba.dim() != 3 or rgba.shape[2] != 4 or not rgba.is_cuda or rgba.dtype != want or not rgba.is_contiguous():
        raise ValueError(f"frame must be a contiguous CUDA {want} tensor [h, w, 4]")
    L = lib()
    h, w = int(rgba.shape[0]), int(rgba.shape[1])
    nbytes = L.pe_yuv420p10_bytes(w, h)
    if nbytes == 0:
        raise PortalB200Error(f"pe_yuv420p10_bytes: no planes for a {w} x {h} frame")
    out = torch.empty(nbytes // 2, dtype=torch.int16, device=rgba.device)
    stream = C.c_void_p(torch.cuda.current_stream(rgba.device).cuda_stream)
    host = np.empty(nbytes // 2, np.uint16)
    if (L.pe_rgba_to_yuv420p10(ctx, C.c_void_p(rgba.data_ptr()), bits, w, h, C.c_void_p(out.data_ptr()), stream)
            or L.pe_memcpy_d2h(ctx, host.ctypes.data, C.c_void_p(out.data_ptr()), nbytes, stream)):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    return yuv420p10_planes(host, w, h)


def yuv420_to_rgba8_device(ctx, yuv, fmt, width: int, height: int):
    """RGBA8 [h, w, 4] (a CUDA uint8 tensor) of the Y'CbCr 4:2:0 planes in the contiguous CUDA tensor `yuv` (uint8 at 8 bits,
    uint16 / int16 at 10; pe_yuv420_bytes long), converted on the device by pe_yuv420_to_rgba8 (DESIGN.md section 5.5) on
    context `ctx`, ordered after the work already queued on the current torch stream.  `fmt`: PeYuvFormat or
    (bits, matrix, full_range, siting)."""
    import torch
    f = yuv_format(fmt)
    L = lib()
    nbytes = L.pe_yuv420_bytes(width, height, f.bits)
    if nbytes == 0:
        raise PortalB200Error(f"pe_yuv420_bytes: no planes for a {width} x {height} frame at {f.bits} bits")
    if not yuv.is_cuda or not yuv.is_contiguous() or yuv.numel() * yuv.element_size() < nbytes:
        raise ValueError(f"planes must be a contiguous CUDA tensor of at least {nbytes} bytes")
    out = torch.empty((height, width, 4), dtype=torch.uint8, device=yuv.device)
    stream = C.c_void_p(torch.cuda.current_stream(yuv.device).cuda_stream)
    if L.pe_yuv420_to_rgba8(ctx, C.c_void_p(yuv.data_ptr()), C.byref(f), width, height, C.c_void_p(out.data_ptr()), stream):
        raise PortalB200Error(L.pe_last_error(ctx).decode(errors="replace"))
    return out
