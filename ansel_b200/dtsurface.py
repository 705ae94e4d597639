"""ctypes mirror of ansel_b200/iop/dt_surface.h so tests and bench.py can call the C module
adapters (dt_iop_<op>__process / __process_cl / __tiling_callback) and the device-resident chain
(b200_pixelpipe_process_on_gpu) the way lib_ansel would."""
from __future__ import annotations

import ctypes as C
import os

from . import MODLIB_PATH, Roi, Tiling, lib as _cuda_lib


class BufferDsc(C.Structure):
    """dt_iop_buffer_dsc_t (src/pixel/format.h:80-119); explicit padding reproduces the 16-byte
    alignment of the two dt_aligned_pixel_t members."""
    _fields_ = [("channels", C.c_uint), ("datatype", C.c_int), ("bpp", C.c_size_t), ("filters", C.c_uint32),
                ("xtrans", C.c_uint8 * 36), ("raw_black_level", C.c_uint16), ("raw_white_point", C.c_uint16),
                ("_pad0", C.c_uint8 * 4), ("temperature_enabled", C.c_int), ("_pad1", C.c_uint8 * 12),
                ("temperature_coeffs", C.c_float * 4), ("processed_maximum", C.c_float * 4), ("cst", C.c_int),
                ("_pad2", C.c_uint8 * 12)]


class Image(C.Structure):
    _fields_ = [("exif_iso", C.c_float), ("flags", C.c_uint32)]


class Develop(C.Structure):
    _fields_ = [("image_storage", Image), ("gui_attached", C.c_int)]


class ProfileInfo(C.Structure):
    """dt_iop_order_iccprofile_info_t subset (src/colorprofiles/iop_profile.h:122-146)."""
    _fields_ = [("matrix_in", (C.c_float * 4) * 3), ("matrix_out", (C.c_float * 4) * 3)]


class Pipe(C.Structure):
    """dt_dev_pixelpipe_t subset."""
    _fields_ = [("dev", C.POINTER(Develop)), ("type", C.c_int), ("mask_display", C.c_int), ("devid", C.c_int),
                ("iscale", C.c_float), ("stream", C.c_void_p), ("work_profile_info", C.POINTER(ProfileInfo)),
                ("output_profile_info", C.POINTER(ProfileInfo)), ("levels", C.c_int)]


class Module(C.Structure):
    _fields_ = [("op", C.c_char * 20), ("dev", C.POINTER(Develop)), ("global_data", C.c_void_p)]


class PipeIop(C.Structure):
    """dt_dev_pixelpipe_iop_t subset (src/develop/pixelpipe_hb.h:101-166)."""
    _fields_ = [("module", C.POINTER(Module)), ("data", C.c_void_p), ("data_size", C.c_size_t), ("enabled", C.c_int),
                ("buf_in", Roi), ("buf_out", Roi), ("roi_in", Roi), ("roi_out", Roi), ("process_cl_ready", C.c_int),
                ("process_tiling_ready", C.c_int), ("_pad_dsc", C.c_uint8 * 8),
                ("dsc_in", BufferDsc), ("dsc_out", BufferDsc)]


PROCESS_CL = C.CFUNCTYPE(C.c_int, C.POINTER(Module), C.POINTER(Pipe), C.POINTER(PipeIop), C.c_void_p, C.c_void_p)


class PipeNode(C.Structure):
    _fields_ = [("process_cl", C.c_void_p), ("module", C.POINTER(Module)), ("piece", C.POINTER(PipeIop)),
                ("blend", C.c_void_p), ("d_form_mask", C.c_void_p), ("d_mask", C.c_void_p)]   # blending: b200_blend_params_t * or NULL


_mod = None
ADAPTED_OPS = ("demosaic", "colorin", "colorout", "denoiseprofile", "filmicrgb", "bilat", "diffuse", "nlmeans",
               "rawprepare", "temperature", "highlights", "exposure", "gamma", "finalscale", "channelmixerrgb", "initialscale", "flip",
               "dither", "lens", "colorbalancergb")


def modlib() -> C.CDLL:
    global _mod
    if _mod is None:
        _cuda_lib()  # libb200iop.so first: the adapters link against it
        if not os.path.exists(MODLIB_PATH):
            raise ImportError(f"{MODLIB_PATH} is missing: run `python -m ansel_b200.build`")
        M = C.CDLL(MODLIB_PATH)
        M.b200_dt_surface_probe.restype = C.c_size_t
        M.b200_pipe_buffers_new.restype = C.c_void_p
        M.b200_pipe_buffers_free.argtypes = [C.c_void_p]
        M.b200_pixelpipe_process_on_gpu.argtypes = [C.POINTER(Pipe), C.POINTER(PipeNode), C.c_int, C.c_void_p,
                                                    C.c_void_p, C.c_void_p]
        M.b200_pipe_queue_new.restype = C.c_void_p
        M.b200_pipe_queue_new.argtypes = [C.c_int]
        M.b200_pipe_queue_free.argtypes = [C.c_void_p]
        M.b200_pixelpipe_submit.restype = C.c_long
        M.b200_pixelpipe_submit.argtypes = [C.c_void_p, C.POINTER(Pipe), C.POINTER(PipeNode), C.c_int, C.c_void_p, C.c_void_p]
        M.b200_pixelpipe_wait.argtypes = [C.c_void_p, C.c_long]
        for op in ADAPTED_OPS:
            getattr(M, f"dt_iop_{op}__process").argtypes = [C.POINTER(Module), C.POINTER(Pipe), C.POINTER(PipeIop),
                                                            C.c_void_p, C.c_void_p]
            getattr(M, f"dt_iop_{op}__process_cl").argtypes = [C.POINTER(Module), C.POINTER(Pipe), C.POINTER(PipeIop),
                                                               C.c_void_p, C.c_void_p]
            getattr(M, f"dt_iop_{op}__tiling_callback").argtypes = [C.POINTER(Module), C.POINTER(Pipe),
                                                                    C.POINTER(PipeIop), C.POINTER(Tiling)]
            getattr(M, f"dt_iop_{op}__tiling_callback").restype = None
        # the ctypes mirror must agree with the C compiler's layout
        assert M.b200_dt_surface_probe(0) == C.sizeof(BufferDsc), "dt_iop_buffer_dsc_t layout"
        assert M.b200_dt_surface_probe(1) == BufferDsc.temperature_coeffs.offset
        assert M.b200_dt_surface_probe(2) == BufferDsc.processed_maximum.offset
        assert M.b200_dt_surface_probe(4) == C.sizeof(PipeIop), "dt_dev_pixelpipe_iop_t layout"
        assert M.b200_dt_surface_probe(6) == PipeIop.dsc_in.offset
        assert M.b200_dt_surface_probe(8) == C.sizeof(Pipe)
        assert M.b200_dt_surface_probe(9) == C.sizeof(Module)
        assert M.b200_dt_surface_probe(12) == C.sizeof(ProfileInfo)
        assert M.b200_dt_surface_probe(13) == Pipe.work_profile_info.offset
        _mod = M
    return _mod


def profile_info(matrix_in, matrix_out) -> ProfileInfo:
    """rows of a dt_colormatrix_t (3x4, last column padding)."""
    import numpy as np
    pi = ProfileInfo()
    for name, m in (("matrix_in", matrix_in), ("matrix_out", matrix_out)):
        m = np.asarray(m, np.float32)
        for r in range(3):
            for c in range(3):
                getattr(pi, name)[r][c] = float(m[r, c])
    return pi


def make_pipe(devid: int = 0, pipe_type: int = 1, stream: int | None = None, exif_iso: float = 100.0, work_profile=None,
              output_profile=None, levels: int = 0x100) -> Pipe:
    """levels: dt_imageio_levels_t of the export (IMAGEIO_RGB | IMAGEIO_INT8 by default)"""
    dev = Develop()
    dev.image_storage.exif_iso = exif_iso
    p = Pipe()
    p._keepalive = dev  # noqa
    p.dev = C.pointer(dev)
    p.type = pipe_type
    p.mask_display = 0
    p.devid = devid
    p.iscale = 1.0
    p.stream = stream
    p.levels = levels
    p._profiles = (work_profile, output_profile)  # noqa
    if work_profile is not None:
        p.work_profile_info = C.pointer(work_profile)
    if output_profile is not None:
        p.output_profile_info = C.pointer(output_profile)
    return p


def make_piece_iop(op: str, width: int, height: int, data, *, channels_in: int, channels_out: int,
                   filters: int = 0, processed_maximum=(1.0, 1.0, 1.0, 1.0), wb=(2.0, 1.0, 1.5, 0.0),
                   type_in: int = 1, type_out: int = 1) -> PipeIop:
    """type_in / type_out: dt_iop_buffer_type_t of the two cachelines (1 float, 2 uint16, 3 uint8)"""
    m = Module()
    m.op = op.encode()
    piece = PipeIop()
    piece._keepalive = (m, data)  # noqa
    piece.module = C.pointer(m)
    if data is not None:
        piece.data = C.cast(C.pointer(data), C.c_void_p)
        piece.data_size = C.sizeof(data)
    piece.enabled = 1
    roi = Roi(0, 0, width, height, 1.0)
    piece.buf_in = piece.buf_out = piece.roi_in = piece.roi_out = roi
    piece.process_cl_ready = 1
    piece.process_tiling_ready = 1
    for dsc, ch, ty in ((piece.dsc_in, channels_in, type_in), (piece.dsc_out, channels_out, type_out)):
        dsc.channels = ch
        dsc.datatype = ty
        dsc.bpp = {1: 4, 2: 2, 3: 1}[ty] * ch
        dsc.filters = filters if ch == 1 else 0
        for k in range(4):
            dsc.processed_maximum[k] = processed_maximum[k]
            dsc.temperature_coeffs[k] = wb[k]
    return piece
