"""ctypes mirror of the C ABI declared in include/ultrahdr_api.h (which itself mirrors the
reference's ultrahdr_api.h:106-283 enums / PODs).  Shared by the product bindings, the tests and
bench.py; holds declarations only, no compute."""
import ctypes as C

import numpy as np

# uhdr_img_fmt_t
FMT_P010, FMT_YUV420, FMT_Y400, FMT_RGBA8888, FMT_RGBAF16, FMT_RGBA1010102 = 0, 1, 2, 3, 4, 5
FMT_YUV444, FMT_YUV422, FMT_RGB888, FMT_YUV444_10 = 6, 7, 11, 12
# uhdr_color_gamut_t
CG_UNSPEC, CG_BT709, CG_P3, CG_BT2100 = -1, 0, 1, 2
# uhdr_color_transfer_t
CT_UNSPEC, CT_LINEAR, CT_HLG, CT_PQ, CT_SRGB = -1, 0, 1, 2, 3
# uhdr_color_range_t
CR_UNSPEC, CR_LIMITED, CR_FULL = -1, 0, 1
# uhdr_img_label_t
HDR_IMG, SDR_IMG, BASE_IMG, GAIN_MAP_IMG = 0, 1, 2, 3
# uhdr_enc_preset_t
USAGE_REALTIME, USAGE_BEST_QUALITY = 0, 1
CODEC_OK = 0

FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)


class ErrorInfo(C.Structure):
    _fields_ = [("error_code", C.c_int), ("has_detail", C.c_int), ("detail", C.c_char * 256)]


class RawImage(C.Structure):
    _fields_ = [("fmt", C.c_int), ("cg", C.c_int), ("ct", C.c_int), ("range", C.c_int),
                ("w", C.c_uint), ("h", C.c_uint), ("planes", C.c_void_p * 3),
                ("stride", C.c_uint * 3)]


class CompressedImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_sz", C.c_size_t), ("capacity", C.c_size_t),
                ("cg", C.c_int), ("ct", C.c_int), ("range", C.c_int)]


class MemBlock(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_sz", C.c_size_t), ("capacity", C.c_size_t)]


class GainmapMetadata(C.Structure):
    _fields_ = [("max_content_boost", C.c_float * 3), ("min_content_boost", C.c_float * 3),
                ("gamma", C.c_float * 3), ("offset_sdr", C.c_float * 3),
                ("offset_hdr", C.c_float * 3), ("hdr_capacity_min", C.c_float),
                ("hdr_capacity_max", C.c_float), ("use_base_cg", C.c_int)]

    def as_dict(self):
        return {k: (list(getattr(self, k)) if hasattr(getattr(self, k), "__len__") else
                    getattr(self, k)) for k, _ in self._fields_}


class GainmapConfig(C.Structure):
    """uhdr_b200_gm_config_t / ref_gm_config: the JpegR constructor arguments
    (lib/include/ultrahdr/ultrahdrcommon.h:450-457) plus generateGainMap's two flags."""
    _fields_ = [("scale_factor", C.c_int), ("quality", C.c_int), ("multichannel", C.c_int),
                ("gamma", C.c_float), ("preset", C.c_int), ("min_content_boost", C.c_float),
                ("max_content_boost", C.c_float), ("target_disp_peak_nits", C.c_float),
                ("sdr_is_601", C.c_int), ("use_luminance", C.c_int)]


def default_gm_config(**kw):
    """Defaults of the C API encoder (ultrahdr_api.cpp:1467-1479): scale 1, q95, multichannel,
    gamma 1, BEST_QUALITY, boosts unset, nits unset; generateGainMap defaults sdr_is_601=false,
    use_luminance=true (lib/include/ultrahdr/ultrahdrcommon.h:496-499)."""
    c = GainmapConfig(1, 95, 1, 1.0, USAGE_BEST_QUALITY, FLT_MIN, FLT_MAX, -1.0, 0, 1)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


SCALE_DENOMS = (1, 2, 4, 8)  # uhdr_b200_decode_scaled_dev / _jpeg_decode_scaled / _scaled_dims: decode at 1/k


def declare_scaled_decode(lib):
    """argument types of the reduced-size decode entry points (include/uhdr_b200.h) on a loaded libuhdr_b200"""
    lib.uhdr_b200_scaled_dims.argtypes = [C.c_void_p, C.c_size_t, C.c_int] + [C.POINTER(C.c_uint)] * 4
    lib.uhdr_b200_decode_scaled_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p]
    lib.uhdr_b200_jpeg_decode_scaled.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data


def raw_image(fmt, cg, ct, rng, w, h, planes, strides):
    """planes: list of numpy arrays (kept alive by the caller)."""
    img = RawImage()
    img.fmt, img.cg, img.ct, img.range, img.w, img.h = fmt, cg, ct, rng, w, h
    for i in range(3):
        img.planes[i] = _ptr(planes[i]) if i < len(planes) else None
        img.stride[i] = strides[i] if i < len(strides) else 0
    return img


def p010_image(buf, w, h, cg, ct, rng, stride=None):
    """buf: uint16 array of w*h*3/2 elements (Y plane then interleaved UV)."""
    stride = stride or w
    y = buf[: stride * h]
    uv = buf[stride * h:]
    img = raw_image(FMT_P010, cg, ct, rng, w, h, [y, uv], [stride, stride])
    return img, (y, uv)


def yuv420_image(buf, w, h, cg, ct=CT_SRGB, rng=CR_FULL):
    y = buf[: w * h]
    u = buf[w * h: w * h + (w // 2) * (h // 2)]
    v = buf[w * h + (w // 2) * (h // 2):]
    img = raw_image(FMT_YUV420, cg, ct, rng, w, h, [y, u, v], [w, w // 2, w // 2])
    return img, (y, u, v)
