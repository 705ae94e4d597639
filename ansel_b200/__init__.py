"""ansel_b200 -- thin Python plumbing over libb200iop.so (the C ABI in include/b200iop.h).

The product is the C-ABI CUDA library plus the C module adapters in ansel_b200/iop/; this package
only loads them (ctypes) so tests and bench.py can drive the same entry points a reference
maintainer would bind from C.  There is no CPU or PyTorch fallback: if the library is missing or
no sm_90 device is present, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200IOP_LIB") or os.path.join(HERE, "libb200iop.so")  # override: development A/B builds only
MODLIB_PATH = os.path.join(HERE, "libb200_modules.so")

# ---- error codes (include/b200iop.h) --------------------------------------------------------
B200_OK, B200_ERR_CUDA, B200_ERR_ARG, B200_ERR_UNSUPPORTED, B200_ERR_NODEVICE, B200_ERR_NOMEM = range(6)

PIPE_NONE, PIPE_EXPORT, PIPE_FULL, PIPE_PREVIEW, PIPE_THUMBNAIL = range(5)

DEMOSAIC_PPG, DEMOSAIC_AMAZE, DEMOSAIC_VNG4, DEMOSAIC_RCD, DEMOSAIC_LMMSE = 0, 1, 2, 5, 6
DEMOSAIC_MARKESTEIJN_3_VNG = 3074  # DT_IOP_DEMOSAIC_MARKEST3_VNG: X-Trans Markesteijn 3-pass + VNG, iop/demosaic.c:138
DEMOSAIC_FDC = 1028  # DT_IOP_DEMOSAIC_FDC: X-Trans frequency-domain chroma, iop/demosaic.c:137 (piece->data: a DemosaicPiece)
DT_IMAGE_4BAYER = 1 << 14  # b200_piece_t.image_flags of a four-colour Bayer sensor (CYGM, RGBE), common/image.h
GREEN_EQ_NO, GREEN_EQ_LOCAL, GREEN_EQ_FULL, GREEN_EQ_BOTH = 0, 1, 2, 3  # dt_iop_demosaic_greeneq_t, iop/demosaic.c:146-149


class Roi(C.Structure):
    """b200_roi_t == dt_iop_roi_t (src/pixel/format.h:48-52)."""
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("width", C.c_int), ("height", C.c_int), ("scale", C.c_double)]


class Tiling(C.Structure):
    """b200_tiling_t == dt_develop_tiling_t (src/develop/tiling.h:39-58)."""
    _fields_ = [("factor", C.c_float), ("factor_cl", C.c_float), ("maxbuf", C.c_float), ("maxbuf_cl", C.c_float),
                ("overhead", C.c_uint), ("overlap", C.c_uint), ("xalign", C.c_uint), ("yalign", C.c_uint)]


class Piece(C.Structure):
    """b200_piece_t: the fields the hot-path process() bodies read (SURVEY.md appendix D)."""
    _fields_ = [("roi_in", Roi), ("roi_out", Roi), ("filters", C.c_uint32), ("xtrans", (C.c_uint8 * 6) * 6),
                ("channels", C.c_uint32), ("processed_maximum", C.c_float * 4), ("wb_coeffs", C.c_float * 4),
                ("buf_in_width", C.c_int), ("buf_in_height", C.c_int), ("pipe_type", C.c_int),
                ("mask_display", C.c_int), ("iscale", C.c_double), ("exif_iso", C.c_float),
                ("image_flags", C.c_uint32), ("devid", C.c_int), ("datatype", C.c_int), ("data", C.c_void_p),
                ("data_size", C.c_size_t)]


class DemosaicData(C.Structure):
    """b200_demosaic_data_t == dt_iop_demosaic_data_t (src/iop/demosaic.c:238-247)."""
    _fields_ = [("green_eq", C.c_uint32), ("color_smoothing", C.c_uint32), ("demosaicing_method", C.c_uint32),
                ("lmmse_refine", C.c_uint32), ("median_thrs", C.c_float), ("CAM_to_RGB", (C.c_double * 4) * 3),
                ("dual_thrs", C.c_float)]


class DemosaicPiece(C.Structure):
    """b200_demosaic_piece_t: the data block + the user's FDC crossover ISO (plugins/darkroom/demosaic/fdc_xover_iso, default 1600)."""
    _fields_ = [("data", DemosaicData), ("fdc_xover_iso", C.c_int)]


LUT_SAMPLES = 0x10000
COLORSPACE_LAB = 6
FP_CONTRACT, FP_STRICT = 0, 1


class Conversion(C.Structure):
    """b200_conversion_t: what a device kernel needs from dt_colorspaces_conversion_t
    (src/colorprofiles/conversion.c:58-97)."""
    _fields_ = [("is_matrix", C.c_int), ("has_clipping", C.c_int), ("matrix", (C.c_float * 4) * 3),
                ("clip_matrix", (C.c_float * 4) * 3), ("lut_source", C.c_void_p * 3),
                ("coeffs_source", (C.c_float * 3) * 3), ("lut_target", C.c_void_p * 3),
                ("coeffs_target", (C.c_float * 3) * 3), ("identity", C.c_uint64), ("fp_mode", C.c_int)]


class ColorinData(C.Structure):
    """b200_colorin_data_t (fields of dt_iop_colorin_data_t, src/iop/colorin.c:145-163)."""
    _fields_ = [("conversion", C.POINTER(Conversion)), ("type", C.c_int), ("blue_mapping", C.c_int)]


class ColoroutData(C.Structure):
    """b200_colorout_data_t (fields of dt_iop_colorout_data_t, src/iop/colorout.c:94-113)."""
    _fields_ = [("conversion", C.POINTER(Conversion)), ("type", C.c_int)]


DENOISE_BANDS = 7
DENOISE_NLMEANS, DENOISE_WAVELETS, DENOISE_VARIANCE, DENOISE_NLMEANS_AUTO, DENOISE_WAVELETS_AUTO = range(5)
DENOISE_RGB, DENOISE_Y0U0V0 = 0, 1


class DenoiseProfileData(C.Structure):
    """b200_denoiseprofile_data_t (members of dt_iop_denoiseprofile_data_t, src/iop/denoiseprofile.c:352-371)."""
    _fields_ = [("radius", C.c_float), ("nbhood", C.c_float), ("strength", C.c_float), ("shadows", C.c_float),
                ("bias", C.c_float), ("scattering", C.c_float), ("central_pixel_weight", C.c_float),
                ("overshooting", C.c_float), ("a", C.c_float * 3), ("b", C.c_float * 3), ("mode", C.c_int),
                ("force", (C.c_float * DENOISE_BANDS) * 6), ("wb_adaptive_anscombe", C.c_int),
                ("fix_anscombe_and_nlmeans_norm", C.c_int), ("use_new_vst", C.c_int), ("wavelet_color_mode", C.c_int)]


FILMIC_DATA_BYTES = 832  # sizeof(dt_iop_filmicrgb_data_t) == sizeof(b200_filmicrgb_data_t)


class FilmicPiece(C.Structure):
    """b200_filmicrgb_piece_t: dt_iop_filmicrgb_data_t (opaque, as commit_params left it) + the work and
    output profile matrices process() fetches from the pipe.  Must live at a 64-byte aligned address."""
    _fields_ = [("data", C.c_uint8 * FILMIC_DATA_BYTES), ("work_in", (C.c_float * 4) * 3), ("work_out", (C.c_float * 4) * 3),
                ("has_export_profile", C.c_int), ("export_in", (C.c_float * 4) * 3), ("export_out", (C.c_float * 4) * 3),
                ("_pad", C.c_uint8 * 60)]


class BilatData(C.Structure):
    """b200_bilat_data_t == dt_iop_bilat_data_t (src/iop/bilat.c:78-86,108)."""
    _fields_ = [("mode", C.c_int), ("sigma_r", C.c_float), ("sigma_s", C.c_float), ("detail", C.c_float), ("midtone", C.c_float)]


class DiffuseData(C.Structure):
    """b200_diffuse_data_t == dt_iop_diffuse_params_t (src/iop/diffuse.c:76-109)."""
    _fields_ = [("iterations", C.c_int), ("sharpness", C.c_float), ("radius", C.c_int), ("regularization", C.c_float),
                ("variance_threshold", C.c_float), ("anisotropy_first", C.c_float), ("anisotropy_second", C.c_float),
                ("anisotropy_third", C.c_float), ("anisotropy_fourth", C.c_float), ("threshold", C.c_float), ("first", C.c_float),
                ("second", C.c_float), ("third", C.c_float), ("fourth", C.c_float), ("radius_center", C.c_int)]


class NlmeansData(C.Structure):
    """b200_nlmeans_data_t == dt_iop_nlmeans_params_t (src/iop/nlmeans.c:81-88)."""
    _fields_ = [("radius", C.c_float), ("strength", C.c_float), ("luma", C.c_float), ("chroma", C.c_float)]


class ProfileMatrices(C.Structure):
    """b200_profile_matrices_t: rows of dt_colormatrix_t (3x4)."""
    _fields_ = [("matrix_in", (C.c_float * 4) * 3), ("matrix_out", (C.c_float * 4) * 3)]


class ProfileCurves(C.Structure):
    """b200_profile_curves_t: tone curves of a matrix profile (lut_in / lut_out, 65536 floats each, host memory)."""
    _fields_ = [("lut_in", C.POINTER(C.c_float) * 3), ("lut_out", C.POINTER(C.c_float) * 3),
                ("unbounded_coeffs_in", (C.c_float * 3) * 3), ("unbounded_coeffs_out", (C.c_float * 3) * 3), ("identity", C.c_uint64)]


TYPE_UNKNOWN, TYPE_FLOAT, TYPE_UINT16, TYPE_UINT8 = range(4)
HIGHLIGHTS_CLIP, HIGHLIGHTS_LCH, HIGHLIGHTS_INPAINT, HIGHLIGHTS_LAPLACIAN, HIGHLIGHTS_HARMONIC = range(5)
EXPORT_UINT8, EXPORT_UINT8_SWAP, EXPORT_UINT16 = range(3)
INTERPOLATION_BILINEAR, INTERPOLATION_BICUBIC, INTERPOLATION_MITCHELL = range(3)


class DngGainMap(C.Structure):
    """b200_dng_gain_map_t header == dt_dng_gain_map_t (src/common/dng_opcode.h:37-55); map_gain[] follows it."""
    _fields_ = [("top", C.c_uint32), ("left", C.c_uint32), ("bottom", C.c_uint32), ("right", C.c_uint32), ("plane", C.c_uint32),
                ("planes", C.c_uint32), ("row_pitch", C.c_uint32), ("col_pitch", C.c_uint32), ("map_points_v", C.c_uint32),
                ("map_points_h", C.c_uint32), ("map_spacing_v", C.c_double), ("map_spacing_h", C.c_double),
                ("map_origin_v", C.c_double), ("map_origin_h", C.c_double), ("map_planes", C.c_uint32)]


class RawprepareData(C.Structure):
    """b200_rawprepare_data_t == dt_iop_rawprepare_data_t (src/iop/rawprepare.c:94-111)."""
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("sub", C.c_float * 4),
                ("div", C.c_float * 4), ("raw_black_level", C.c_uint16), ("raw_white_point", C.c_uint16),
                ("apply_gainmaps", C.c_int), ("gainmaps", C.c_void_p * 4)]


class TemperatureData(C.Structure):
    """b200_temperature_data_t == dt_iop_temperature_data_t (src/iop/temperature.c:150-153)."""
    _fields_ = [("coeffs", C.c_float * 4)]


class HighlightsData(C.Structure):
    """b200_highlights_data_t == dt_iop_highlights_params_t (src/iop/highlights/common.h:456-476)."""
    _fields_ = [("mode", C.c_int), ("blendL", C.c_float), ("blendC", C.c_float), ("blendh", C.c_float), ("clip", C.c_float),
                ("noise_level", C.c_float), ("iterations", C.c_int), ("scales", C.c_int), ("reconstructing", C.c_float),
                ("combine", C.c_float), ("debugmode", C.c_int), ("solid_color", C.c_float)]


class ExposureData(C.Structure):
    """b200_exposure_data_t == dt_iop_exposure_data_t (src/iop/exposure.c:116-124,151-157)."""
    _fields_ = [("mode", C.c_int), ("p_black", C.c_float), ("p_exposure", C.c_float), ("deflicker_percentile", C.c_float),
                ("deflicker_target_level", C.c_float), ("compensate_exposure_bias", C.c_int), ("deflicker", C.c_int),
                ("black", C.c_float), ("scale", C.c_float)]


class FinalscaleData(C.Structure):
    """b200_finalscale_data_t: dt_iop_finalscale_data_t's dummy int + the user-preference interpolator the adapter resolves."""
    _fields_ = [("dummy", C.c_int), ("interpolator", C.c_int)]


ADAPTATION_LINEAR_BRADFORD, ADAPTATION_CAT16, ADAPTATION_FULL_BRADFORD, ADAPTATION_XYZ, ADAPTATION_RGB = range(5)


class ChannelmixerPiece(C.Structure):
    """b200_channelmixerrgb_piece_t: dt_iop_channelmixer_rbg_data_t (src/iop/channelmixerrgb.c:259-272; 64-byte aligned, 192 bytes)
    + the work profile's matrices process() fetches.  Must live at a 64-byte aligned address (channelmixer_piece())."""
    _fields_ = [("MIX", (C.c_float * 4) * 4), ("saturation", C.c_float * 4), ("lightness", C.c_float * 4), ("grey", C.c_float * 4),
                ("illuminant", C.c_float * 4), ("p", C.c_float), ("gamut", C.c_float), ("apply_grey", C.c_int), ("clip", C.c_int),
                ("adaptation", C.c_int), ("illuminant_type", C.c_int), ("version", C.c_int), ("_pad0", C.c_uint8 * 36),
                ("work_in", (C.c_float * 4) * 3), ("work_out", (C.c_float * 4) * 3), ("_pad1", C.c_uint8 * 32)]


class FlipData(C.Structure):
    """b200_flip_data_t == dt_iop_flip_params_t (src/iop/flip.c:74-79): dt_image_orientation_t."""
    _fields_ = [("orientation", C.c_int)]


DITHER_RANDOM, DITHER_FS1BIT, DITHER_FS4BIT_GRAY, DITHER_FS8BIT, DITHER_FS16BIT, DITHER_FSAUTO = range(6)
IMAGEIO_INT8, IMAGEIO_INT12, IMAGEIO_INT16, IMAGEIO_INT32, IMAGEIO_FLOAT, IMAGEIO_BW = range(6)
IMAGEIO_PREC_MASK, IMAGEIO_RGB, IMAGEIO_GRAY, IMAGEIO_CHANNEL_MASK = 0xFF, 0x100, 0x200, 0xFF00


class DitherData(C.Structure):
    """b200_dither_data_t: dt_iop_dither_data_t (src/iop/dither.c:104-113) + pipe->levels (dt_imageio_levels_t), which the adapter fills."""
    _fields_ = [("dither_type", C.c_int), ("radius", C.c_float), ("range", C.c_float * 4), ("damping", C.c_float), ("levels", C.c_int)]


LENS_MODIFY_TCA, LENS_MODIFY_VIGNETTING, LENS_MODIFY_DISTORTION, LENS_MODIFY_GEOMETRY, LENS_MODIFY_SCALE = 0x01, 0x02, 0x08, 0x10, 0x20
LS_DIST_NONE, LS_DIST_POLY3, LS_DIST_POLY5, LS_DIST_PTLENS, LS_DIST_KNOTS = range(5)
LS_TCA_NONE, LS_TCA_LINEAR, LS_TCA_POLY3 = range(3)
LS_VIG_NONE, LS_VIG_PA, LS_VIG_KNOTS = range(3)
(LENS_UNKNOWN, LENS_RECTILINEAR, LENS_FISHEYE, LENS_PANORAMIC, LENS_EQUIRECTANGULAR, LENS_FISHEYE_ORTHOGRAPHIC,
 LENS_FISHEYE_STEREOGRAPHIC, LENS_FISHEYE_EQUISOLID, LENS_FISHEYE_THOBY) = range(9)
LS_ENABLE_DISTORTION, LS_ENABLE_TCA, LS_ENABLE_VIGNETTING, LS_ENABLE_SCALE, LS_ENABLE_GEOMETRY = 1, 2, 4, 8, 16
IMAGE_MONOCHROME, IMAGE_MONOCHROME_BAYER = 1 << 15, 1 << 19
LS_MAX_CALIB, LS_MAX_KNOTS = 512, 16


class LsCalibDist(C.Structure):
    _fields_ = [("model", C.c_int), ("focal", C.c_float), ("terms", C.c_float * 3)]


class LsCalibTca(C.Structure):
    _fields_ = [("model", C.c_int), ("focal", C.c_float), ("terms", C.c_float * 6)]


class LsCalibVig(C.Structure):
    _fields_ = [("model", C.c_int), ("focal", C.c_float), ("aperture", C.c_float), ("distance", C.c_float), ("terms", C.c_float * 3)]


class LsCalibRealFocal(C.Structure):
    _fields_ = [("focal", C.c_float), ("real_focal", C.c_float)]


class LsLens(C.Structure):
    """b200_ls_lens_t == ls_lens_t (src/external/LensSerious/include/lensserious.h:108-129)."""
    _fields_ = [("type", C.c_int), ("crop_factor", C.c_float), ("aspect_ratio", C.c_float), ("min_focal", C.c_float), ("max_focal", C.c_float),
                ("center_x", C.c_float), ("center_y", C.c_float),
                ("n_dist", C.c_int), ("dist", LsCalibDist * LS_MAX_CALIB), ("n_tca", C.c_int), ("tca", LsCalibTca * LS_MAX_CALIB),
                ("n_vig", C.c_int), ("vig", LsCalibVig * LS_MAX_CALIB), ("n_real_focal", C.c_int), ("real_focal", LsCalibRealFocal * LS_MAX_CALIB)]


class LensData(C.Structure):
    """b200_lens_data_t == dt_iop_lensfun_data_t (src/iop/lens.c:392-409)."""
    _fields_ = [("modify_flags", C.c_int), ("inverse", C.c_int), ("scale", C.c_float), ("crop", C.c_float), ("focal", C.c_float),
                ("aperture", C.c_float), ("distance", C.c_float), ("target_geom", C.c_int), ("do_nan_checks", C.c_int),
                ("tca_override", C.c_int), ("ls_lens", LsLens), ("ls_have", C.c_int)]


class LensPiece(C.Structure):
    """b200_lens_piece_t: the data block + the warp interpolator process() resolves from the user preference."""
    _fields_ = [("data", LensData), ("interpolation", C.c_int)]


class LensEval(C.Structure):
    """b200_lens_eval_t == ls_eval_t (src/external/LensSerious/include/lensserious_eval.h:143-194)."""
    _fields_ = [("norm_scale", C.c_float), ("norm_unscale", C.c_float), ("center_x", C.c_float), ("center_y", C.c_float),
                ("vig_scale", C.c_float), ("vig_center_x", C.c_float), ("vig_center_y", C.c_float), ("scale", C.c_float),
                ("dist_model", C.c_int), ("tca_model", C.c_int), ("vig_model", C.c_int), ("enabled", C.c_int), ("geom_from", C.c_int),
                ("geom_to", C.c_int), ("geom_focal", C.c_float), ("reverse", C.c_int), ("dist_terms", C.c_float * 3),
                ("tca_terms", C.c_float * 6), ("vig_terms", C.c_float * 3), ("knot_n", C.c_int),
                ("knot_r", (C.c_float * LS_MAX_KNOTS) * 3), ("knot_c", (C.c_float * LS_MAX_KNOTS) * 3), ("knot_vn", C.c_int),
                ("knot_vr", C.c_float * LS_MAX_KNOTS), ("knot_v", C.c_float * LS_MAX_KNOTS)]


COLORBALANCE_SATURATION_JZAZBZ, COLORBALANCE_SATURATION_DTUCS = 0, 1
COLORBALANCE_LUT_ELEM = 360


class ColorbalancergbData(C.Structure):
    """b200_colorbalancergb_data_t == dt_iop_colorbalancergb_data_t up to work_profile (src/iop/colorbalancergb.c:165-189), 232 bytes."""
    _fields_ = [("global_", C.c_float * 4), ("shadows", C.c_float * 4), ("highlights", C.c_float * 4), ("midtones", C.c_float * 4),
                ("midtones_Y", C.c_float), ("chroma_global", C.c_float), ("chroma", C.c_float * 4), ("vibrance", C.c_float),
                ("contrast", C.c_float), ("saturation_global", C.c_float), ("saturation", C.c_float * 4), ("brilliance_global", C.c_float),
                ("brilliance", C.c_float * 4), ("hue_angle", C.c_float), ("shadows_weight", C.c_float), ("highlights_weight", C.c_float),
                ("midtones_weight", C.c_float), ("mask_grey_fulcrum", C.c_float), ("white_fulcrum", C.c_float), ("grey_fulcrum", C.c_float),
                ("max_chroma", C.c_float), ("checker_color_1", C.c_float * 4), ("checker_color_2", C.c_float * 4),
                ("saturation_formula", C.c_int), ("checker_size", C.c_size_t), ("mask_preview_black_and_white", C.c_int),
                ("mask_display", C.c_int), ("mask_type", C.c_int), ("lut_inited", C.c_int)]


class ColorbalancergbPiece(C.Structure):
    """b200_colorbalancergb_piece_t: the data block, the work profile's matrices and the 360 floats of the gamut LUT."""
    _fields_ = [("data", ColorbalancergbData), ("work_profile", ProfileMatrices), ("gamut_LUT", C.c_float * COLORBALANCE_LUT_ELEM)]


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libb200iop error {code}: {msg}")
        self.code = code


OPS = ("demosaic", "colorin", "colorout", "denoiseprofile", "filmicrgb", "bilat", "diffuse", "nlmeans",
       "rawprepare", "temperature", "highlights", "exposure", "gamma", "finalscale", "channelmixerrgb", "initialscale", "flip", "dither")

_lib = None


def lib() -> C.CDLL:
    """Load libb200iop.so (built in-tree by ansel_b200.build).  Fails loudly when absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -m ansel_b200.build` (needs nvcc)")
        L = C.CDLL(LIB_PATH)
        L.b200_last_error.restype = C.c_char_p
        L.b200_roi_filters.restype = C.c_uint32
        L.b200_roi_filters.argtypes = [C.c_uint32, C.c_int, C.c_int]
        L.b200_fc.argtypes = [C.c_int, C.c_int, C.c_uint32]
        for op in OPS:
            getattr(L, f"b200_{op}_process_host").argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p]
            getattr(L, f"b200_{op}_process_dev").argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p, C.c_void_p]
            getattr(L, f"b200_{op}_tiling").argtypes = [C.POINTER(Piece), C.POINTER(Tiling)]
            getattr(L, f"b200_{op}_tiling").restype = None
        # lens correction (piece->data: a b200_lens_piece_t from lens_piece()) and its host plan
        L.b200_lens_process_host.argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p]
        L.b200_lens_process_dev.argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200_lens_tiling.argtypes = [C.POINTER(Piece), C.POINTER(Tiling)]
        L.b200_lens_tiling.restype = None
        L.b200_lens_plan.argtypes = [C.POINTER(LensData), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(LensEval)]
        # colour balance rgb (piece->data: a b200_colorbalancergb_piece_t from colorbalancergb_piece())
        L.b200_colorbalancergb_process_host.argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p]
        L.b200_colorbalancergb_process_dev.argtypes = [C.POINTER(Piece), C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200_colorbalancergb_tiling.argtypes = [C.POINTER(Piece), C.POINTER(Tiling)]
        L.b200_colorbalancergb_tiling.restype = None
        L.b200_highlights_laplacian_dev.argtypes =[C.POINTER(Piece), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200_rawfront_process_dev.argtypes = [C.POINTER(Piece), C.POINTER(Piece), C.POINTER(Piece), C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200_resampling_plan.argtypes = [C.c_int] * 5 + [C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.b200_basebuffer_upload_dev.argtypes = [C.POINTER(Piece), C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.c_void_p]
        L.b200_export_convert_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
        L.b200_export_convert_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]
        L.b200_apply_conversion_dev.argtypes = [C.POINTER(Conversion), C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t,
                                                C.c_int, C.c_void_p]
        L.b200_eaw_dn_decompose_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int,
                                                C.c_int, C.c_void_p]
        L.b200_eaw_synthesize_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p]
        L.b200_nlmeans_denoise_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float,
                                               C.c_float, C.c_float, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.b200_flt32_eval_dev.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.b200_fit_unbounded_coeffs.argtypes = [C.POINTER(C.c_void_p), C.c_void_p]
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode("utf-8", "replace"))


def init(ndev: int = 0) -> int:
    check(lib().b200_init(ndev))
    return lib().b200_device_count()


def make_piece(width: int, height: int, *, filters: int = 0x94949494, roi_x: int = 0, roi_y: int = 0,
               processed_maximum=(1.0, 1.0, 1.0, 1.0), wb_coeffs=(2.0, 1.0, 1.5, 0.0), channels: int = 1,
               pipe_type: int = PIPE_EXPORT, exif_iso: float = 100.0, devid: int = -1, data=None,
               out_width: int | None = None, out_height: int | None = None, scale: float = 1.0) -> Piece:
    """Fill a b200_piece_t with the fixed metadata of SURVEY.md 8(d)."""
    p = Piece()
    p.roi_in = Roi(roi_x, roi_y, width, height, scale)
    p.roi_out = Roi(0, 0, out_width or width, out_height or height, scale)
    p.filters = filters
    p.channels = channels
    for k in range(4):
        p.processed_maximum[k] = processed_maximum[k] if k < len(processed_maximum) else 0.0
        p.wb_coeffs[k] = wb_coeffs[k] if k < len(wb_coeffs) else 0.0
    p.buf_in_width, p.buf_in_height = width, height
    p.pipe_type = pipe_type
    p.mask_display = 0
    p.iscale = 1.0
    p.exif_iso = exif_iso
    p.image_flags = 0
    p.devid = devid
    if data is not None:
        p._keepalive = data  # noqa: keep the ctypes struct alive with the piece
        p.data = C.cast(C.pointer(data), C.c_void_p)
        p.data_size = C.sizeof(data)
    return p


def demosaic_data(method: int = DEMOSAIC_RCD) -> DemosaicData:
    d = DemosaicData()
    d.demosaicing_method = method
    return d


def make_conversion(matrix, *, clip_matrix=None, lut_source=None, coeffs_source=None, lut_target=None,
                    coeffs_target=None, identity: int = 0, fp_mode: int = FP_CONTRACT) -> Conversion:
    """Fill a b200_conversion_t from numpy arrays (3x3 matrices, 3 x LUT_SAMPLES float32 curves).
    The arrays are kept alive on the returned struct."""
    import numpy as np
    c = Conversion()
    c.is_matrix = 1
    c.has_clipping = 1 if clip_matrix is not None else 0
    keep = []
    for i in range(3):
        for j in range(3):
            c.matrix[i][j] = float(matrix[i][j])
            c.clip_matrix[i][j] = float(clip_matrix[i][j]) if clip_matrix is not None else 0.0
            c.coeffs_source[i][j] = float(coeffs_source[i][j]) if coeffs_source is not None else 0.0
            c.coeffs_target[i][j] = float(coeffs_target[i][j]) if coeffs_target is not None else 0.0
    for name, lut in (("lut_source", lut_source), ("lut_target", lut_target)):
        if lut is not None:
            arr = np.ascontiguousarray(lut, dtype=np.float32)
            assert arr.shape == (3, LUT_SAMPLES)
            keep.append(arr)
            for k in range(3):
                getattr(c, name)[k] = arr[k].ctypes.data
    c.identity = identity
    c.fp_mode = fp_mode
    c._keepalive = keep  # noqa
    return c


def colorin_data(conversion: Conversion | None, type_: int = 12) -> ColorinData:
    d = ColorinData()
    if conversion is not None:
        d._keepalive = conversion  # noqa
        d.conversion = C.pointer(conversion)
    d.type = type_
    return d


def colorout_data(conversion: Conversion | None, type_: int = 1) -> ColoroutData:
    d = ColoroutData()
    if conversion is not None:
        d._keepalive = conversion  # noqa
        d.conversion = C.pointer(conversion)
    d.type = type_
    return d


def infer_shadows_from_profile(a: float) -> float:
    """iop/denoiseprofile.c:2659-2662."""
    import math
    import numpy as np
    return float(min(max(0.1 - 0.1 * float(np.log(np.float32(a))), 0.7), 1.8))


def infer_bias_from_profile(a: float) -> float:
    """iop/denoiseprofile.c:2664-2667."""
    import numpy as np
    return float(-max(5 + 0.5 * float(np.log(np.float32(a))), 0.0))


def denoiseprofile_data(mode: int = DENOISE_WAVELETS, *, a=(1e-4, 1e-4, 1e-4), b=(0.0, 0.0, 0.0), strength: float = 1.0,
                        radius: float = 1.0, nbhood: float = 7.0, scattering: float = 0.0,
                        central_pixel_weight: float = 0.1, color_mode: int = DENOISE_Y0U0V0, force: float = 0.5,
                        use_new_vst: bool = True, shadows: float | None = None, bias: float | None = None) -> DenoiseProfileData:
    """Parameters of SURVEY.md 8(d): generic Poissonian profile, shadows/bias inferred from it, flat
    wavelet force curves (the GUI default nodes evaluate to 0.5 on every band)."""
    d = DenoiseProfileData()
    d.radius, d.nbhood, d.strength, d.scattering = radius, nbhood, strength, scattering
    d.central_pixel_weight, d.overshooting = central_pixel_weight, 1.0
    d.shadows = infer_shadows_from_profile(a[1]) if shadows is None else shadows
    d.bias = infer_bias_from_profile(a[1]) if bias is None else bias
    for k in range(3):
        d.a[k], d.b[k] = a[k], b[k]
    d.mode = mode
    for ch in range(6):
        for band in range(DENOISE_BANDS):
            d.force[ch][band] = force
    d.wb_adaptive_anscombe = 1
    d.fix_anscombe_and_nlmeans_norm = 1
    d.use_new_vst = 1 if use_new_vst else 0
    d.wavelet_color_mode = color_mode
    return d


def filmic_piece(data_blob, work, export=None) -> FilmicPiece:
    """data_blob: 832 bytes of dt_iop_filmicrgb_data_t; work/export: (matrix_in, matrix_out) 3x3 arrays."""
    import numpy as np
    assert C.sizeof(FilmicPiece) == 1088
    raw = np.zeros(C.sizeof(FilmicPiece) + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    fp = FilmicPiece.from_buffer(raw, off)
    fp._keepalive = raw  # noqa
    C.memmove(C.addressof(fp), np.ascontiguousarray(data_blob, np.uint8).ctypes.data, FILMIC_DATA_BYTES)
    for dst, src in ((fp.work_in, work[0]), (fp.work_out, work[1])) + (((fp.export_in, export[0]), (fp.export_out, export[1])) if export else ()):
        for i in range(3):
            for j in range(3):
                dst[i][j] = float(src[i][j])
    fp.has_export_profile = 1 if export else 0
    return fp


def bilat_data(sigma_r: float = 0.5, sigma_s: float = 0.5, detail: float = 0.25, midtone: float = 0.5, mode: int = 1) -> BilatData:
    return BilatData(mode, sigma_r, sigma_s, detail, midtone)


# stock presets of src/iop/diffuse.c init_presets(), values as registered there
DIFFUSE_PRESETS = {
    "defaults": dict(),
    # "lens deblur: soft" :298-320
    "lens_deblur_soft": dict(iterations=8, radius=8, regularization=1.0, variance_threshold=0.0, anisotropy_first=2.0,
                             anisotropy_second=0.0, anisotropy_third=2.0, anisotropy_fourth=0.0, first=-0.25, second=0.125,
                             third=-0.125, fourth=0.0625),
    # "sharpen demosaicing (AA filter)" :440-461
    "sharpen_demosaic_aa": dict(iterations=1, radius=8, regularization=1.0, variance_threshold=0.0, anisotropy_first=1.0,
                                anisotropy_second=1.0, anisotropy_third=1.0, anisotropy_fourth=1.0, first=-0.25, second=-0.25,
                                third=-0.25, fourth=-0.25),
    # "denoise: medium" :364-391
    "denoise_medium": dict(iterations=32, radius=3, radius_center=4, regularization=2.5, variance_threshold=-0.0, anisotropy_first=2.0,
                           anisotropy_second=0.0, anisotropy_third=2.0, anisotropy_fourth=0.0, first=0.10, second=0.0, third=0.10,
                           fourth=0.0),
    # "surface blur" :404-420
    "surface_blur": dict(iterations=2, radius=32, regularization=4.0, variance_threshold=0.0, anisotropy_first=4.0, anisotropy_second=4.0,
                         anisotropy_third=4.0, anisotropy_fourth=4.0, first=1.0, second=1.0, third=1.0, fourth=1.0),
    # "bloom" :422-438
    "bloom": dict(iterations=1, radius=32, regularization=0.0, variance_threshold=0.0, first=0.5, second=0.5, third=0.5, fourth=0.5),
    # "inpaint highlights" :518-538: the luminance mask (threshold > 0) with its noise-seeded start image
    "inpaint_highlights": dict(iterations=32, radius=4, radius_center=0, sharpness=0.0, threshold=1.41, variance_threshold=0.0,
                               regularization=0.0, anisotropy_first=0.0, anisotropy_second=0.0, anisotropy_third=0.0,
                               anisotropy_fourth=2.0, first=0.0, second=0.0, third=0.0, fourth=0.5),
}


def diffuse_data(**kw) -> DiffuseData:
    """$DEFAULTs of dt_iop_diffuse_params_t, overridden by keyword."""
    d = DiffuseData(iterations=1, sharpness=0.0, radius=8, regularization=0.0, variance_threshold=0.0, anisotropy_first=0.0,
                    anisotropy_second=0.0, anisotropy_third=0.0, anisotropy_fourth=0.0, threshold=0.0, first=0.0, second=0.0,
                    third=0.0, fourth=0.0, radius_center=0)
    for k, v in kw.items():
        assert hasattr(d, k), k
        setattr(d, k, v)
    return d


CS_LAB, CS_RGB = 1, 2


def nlmeans_data(radius: float = 2.0, strength: float = 50.0, luma: float = 0.5, chroma: float = 1.0) -> NlmeansData:
    return NlmeansData(radius, strength, luma, chroma)


def profile_curves(lut_in, co_in, lut_out, co_out, identity: int = 0) -> ProfileCurves:
    """lut_*: float32 arrays (3, 65536), kept alive on the returned struct; co_*: (3, 3) unbounded coefficients."""
    import numpy as np
    pc = ProfileCurves()
    pc._keep = [np.ascontiguousarray(lut_in, np.float32), np.ascontiguousarray(lut_out, np.float32)]
    for k in range(3):
        pc.lut_in[k] = pc._keep[0][k].ctypes.data_as(C.POINTER(C.c_float))
        pc.lut_out[k] = pc._keep[1][k].ctypes.data_as(C.POINTER(C.c_float))
        for j in range(3):
            pc.unbounded_coeffs_in[k][j] = float(co_in[k][j])
            pc.unbounded_coeffs_out[k][j] = float(co_out[k][j])
    pc.identity = identity
    return pc


def profile_matrices(matrix_in, matrix_out) -> ProfileMatrices:
    pm = ProfileMatrices()
    for name, m in (("matrix_in", matrix_in), ("matrix_out", matrix_out)):
        for r in range(3):
            for c in range(3):
                getattr(pm, name)[r][c] = float(m[r][c])
    return pm


def rawprepare_data(sub, div, x: int = 0, y: int = 0, gain=None, spacing=(0.0, 0.0), origin=(0.0, 0.0)) -> RawprepareData:
    """sub/div: the four per-site black levels and ranges commit_params() leaves (rawprepare.c:722-750); gain: None or a
    float32 array [4, map_h, map_w] (spacing/origin = (h, v), relative to the full image)."""
    import numpy as np
    d = RawprepareData()
    d.x, d.y = x, y
    for k in range(4):
        d.sub[k], d.div[k] = sub[k], div[k]
    if gain is not None:
        gain = np.ascontiguousarray(gain, dtype=np.float32)
        _, mh, mw = gain.shape
        keep = []
        for f in range(4):
            buf = (C.c_uint8 * (C.sizeof(DngGainMap) + 4 + 4 * mw * mh))()  # map_gain[] starts at offsetof == sizeof - padding
            hdr = DngGainMap.from_buffer(buf)
            hdr.map_points_h, hdr.map_points_v = mw, mh
            hdr.map_spacing_h, hdr.map_spacing_v = spacing
            hdr.map_origin_h, hdr.map_origin_v = origin
            C.memmove(C.addressof(buf) + DngGainMap.map_planes.offset + 4, gain[f].ctypes.data, 4 * mw * mh)
            keep.append(buf)
            d.gainmaps[f] = C.addressof(buf)
        d.apply_gainmaps = 1
        d._keepalive = keep
    return d


def temperature_data(coeffs) -> TemperatureData:
    d = TemperatureData()
    for k in range(4):
        d.coeffs[k] = coeffs[k] if k < len(coeffs) else 0.0
    return d


def highlights_data(mode: int = HIGHLIGHTS_CLIP, clip: float = 1.0) -> HighlightsData:
    d = HighlightsData()
    d.mode, d.clip, d.blendL, d.iterations, d.scales, d.reconstructing, d.combine = mode, clip, 1.0, 30, 8, 0.4, 2.0
    return d


def exposure_data(black: float = 0.0, exposure_ev: float = 0.0) -> ExposureData:
    """black/scale as _process_common_setup() derives them (exposure.c:433-470): white = exp2f(-exposure),
    scale = 1.0 / (white - black) with a double division."""
    import numpy as np
    d = ExposureData()
    d.p_black, d.p_exposure, d.deflicker_percentile, d.deflicker_target_level = black, exposure_ev, 50.0, -4.0
    d.black = black
    white = np.exp2(np.float32(-exposure_ev), dtype=np.float32)
    d.scale = float(np.float32(1.0 / float(white - np.float32(black))))
    return d


def finalscale_data(interpolator: int = INTERPOLATION_MITCHELL) -> FinalscaleData:
    d = FinalscaleData()
    d.interpolator = interpolator
    return d


def channelmixer_piece(work, *, adaptation: int = ADAPTATION_CAT16, illuminant=(0.95, 1.0, 0.85), mix=None, saturation=(0.0, 0.0, 0.0),
                       lightness=(0.0, 0.0, 0.0), grey=(0.0, 0.0, 0.0), p: float = 0.9, gamut: float = 1.0, clip: int = 1, apply_grey: int = 0,
                       version: int = 2) -> ChannelmixerPiece:
    """work: (matrix_in, matrix_out) 3x3 arrays of the pipe's work profile; the rest as commit_params() (channelmixerrgb.c:2290-2440)
    leaves it: illuminant in the adaptation's LMS/XYZ space, mix = 3x3 rows (identity by default)."""
    import numpy as np
    assert C.sizeof(ChannelmixerPiece) == 320
    raw = np.zeros(C.sizeof(ChannelmixerPiece) + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    cp = ChannelmixerPiece.from_buffer(raw, off)
    cp._keepalive = raw  # noqa
    mix = np.eye(3, dtype=np.float32) if mix is None else np.asarray(mix, np.float32)
    for i in range(3):
        for j in range(3):
            cp.MIX[i][j] = float(mix[i][j])
            cp.work_in[i][j] = float(work[0][i][j])
            cp.work_out[i][j] = float(work[1][i][j])
        cp.saturation[i], cp.lightness[i], cp.grey[i], cp.illuminant[i] = saturation[i], lightness[i], grey[i], illuminant[i]
    cp.p, cp.gamut, cp.apply_grey, cp.clip, cp.adaptation, cp.version = p, gamut, apply_grey, clip, adaptation, version
    return cp


def dither_data(dither_type: int = DITHER_FSAUTO, levels: int = IMAGEIO_RGB | IMAGEIO_INT8) -> DitherData:
    """the module's defaults (dither.c:154-155: FS auto, damping -200) for an export at `levels`"""
    d = DitherData()
    d.dither_type = dither_type
    d.range[2] = d.range[3] = 1.0
    d.damping = -200.0
    d.levels = levels
    return d


def lens_piece(data: LensData, interpolation: int = INTERPOLATION_MITCHELL) -> LensPiece:
    """b200_lens_piece_t: a copy of the data block + the warp interpolator (the preference's default: Mitchell)"""
    lp = LensPiece()
    C.memmove(C.addressof(lp.data), C.addressof(data), C.sizeof(LensData))
    lp.interpolation = interpolation
    return lp


def colorbalancergb_piece(data_blob, work, lut) -> ColorbalancergbPiece:
    """data_blob: the 232 bytes of dt_iop_colorbalancergb_data_t commit_params() leaves (or a ColorbalancergbData); work: (matrix_in,
    matrix_out) 3x3 arrays of the pipe's work profile; lut: the 360 floats behind data->gamut_LUT."""
    import numpy as np
    assert C.sizeof(ColorbalancergbData) == 232
    cp = ColorbalancergbPiece()
    blob = bytes(data_blob) if isinstance(data_blob, ColorbalancergbData) else np.ascontiguousarray(data_blob, np.uint8).tobytes()
    assert len(blob) == C.sizeof(ColorbalancergbData)
    C.memmove(C.addressof(cp.data), blob, len(blob))
    cp.work_profile = profile_matrices(work[0], work[1])
    lut = np.ascontiguousarray(lut, np.float32)
    assert lut.shape == (COLORBALANCE_LUT_ELEM,)
    C.memmove(C.addressof(cp.gamut_LUT), lut.ctypes.data, lut.nbytes)
    return cp
