"""ctypes binding of lib/libpsb200.so (C-ABI in include/psb200.h). Fails loudly when the library is missing."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libpsb200.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_size_t, C.c_void_p)

_lib = None


class RasterPlanes(C.Structure):
    """psb_raster_planes: the planes psb_rasterize_forward_planes renders beside colour (device pointers; None = not rendered)."""
    _fields_ = [("out_depth", C.c_void_p), ("out_alpha", C.c_void_p), ("out_normal", C.c_void_p), ("out_depth2", C.c_void_p)]


class RasterPlaneGrads(C.Structure):
    """psb_raster_plane_grads: the plane gradients psb_rasterize_backward_planes takes (device pointers; None = no gradient)."""
    _fields_ = [("dL_ddepth", C.c_void_p), ("dL_dalpha", C.c_void_p), ("dL_dnormal", C.c_void_p), ("dL_ddepth2", C.c_void_p)]


class PsbError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PsbError(
            f"{LIB_PATH} not found: build it with `python photo-slam_b200/build.py` "
            "(or __graft_entry__.build()). There is no CPU fallback for the rasterizer.")
    L = C.CDLL(LIB_PATH)
    fp, ip, vp, u8p = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p  # device pointers travel as integers
    L.psb_version.restype = C.c_int
    L.psb_last_error.restype = C.c_char_p
    for name in ("psb_geometry_bytes", "psb_binning_bytes", "psb_image_bytes"):
        getattr(L, name).restype = C.c_size_t
        getattr(L, name).argtypes = [C.c_int]
    L.psb_rasterize_forward.restype = C.c_int
    L.psb_rasterize_forward.argtypes = [
        ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp, C.c_int, C.c_int, C.c_int, fp, C.c_int, C.c_int,
        fp, fp, fp, fp, fp, C.c_float, fp, fp, fp, fp, fp, C.c_float, C.c_float, C.c_int, fp, ip, vp]
    L.psb_rasterize_backward.restype = C.c_int
    L.psb_rasterize_backward.argtypes = [
        C.c_int, C.c_int, C.c_int, C.c_int, fp, C.c_int, C.c_int, fp, fp, fp, fp, C.c_float, fp, fp, fp, fp, fp,
        C.c_float, C.c_float, ip, vp, vp, vp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, vp]
    # the _depth variants: the plain argument list plus out_depth, and plus dL_ddepth, dL_dz, before the stream
    L.psb_rasterize_forward_depth.restype = C.c_int
    L.psb_rasterize_forward_depth.argtypes = L.psb_rasterize_forward.argtypes[:-1] + [fp, vp]
    L.psb_rasterize_backward_depth.restype = C.c_int
    L.psb_rasterize_backward_depth.argtypes = L.psb_rasterize_backward.argtypes[:-1] + [fp, fp, vp]
    # the deterministic backward: the _depth argument list plus det_scratch, det_scratch_bytes, before the stream
    L.psb_rasterize_backward_det_bytes.restype = C.c_size_t
    L.psb_rasterize_backward_det_bytes.argtypes = [C.c_int, C.c_int]
    L.psb_rasterize_backward_deterministic.restype = C.c_int
    L.psb_rasterize_backward_deterministic.argtypes = L.psb_rasterize_backward_depth.argtypes[:-1] + [vp, C.c_size_t, vp]
    # anti-aliasing: the _depth forward's and the deterministic backward's argument lists plus `antialiasing`, before the stream
    L.psb_rasterize_forward_aa.restype = C.c_int
    L.psb_rasterize_forward_aa.argtypes = L.psb_rasterize_forward_depth.argtypes[:-1] + [C.c_int, vp]
    L.psb_rasterize_backward_aa.restype = C.c_int
    L.psb_rasterize_backward_aa.argtypes = L.psb_rasterize_backward_deterministic.argtypes[:-1] + [C.c_int, vp]
    # opacity, normals and the second depth moment: the _aa argument lists with out_depth / dL_ddepth moved into a record (passed by
    # pointer), plus plane_scratch, plane_scratch_bytes (and `deterministic` on the backward)
    L.psb_rasterize_planes_bytes.restype = C.c_size_t
    L.psb_rasterize_planes_bytes.argtypes = [C.c_int, C.c_int]
    L.psb_rasterize_forward_planes.restype = C.c_int
    L.psb_rasterize_forward_planes.argtypes = L.psb_rasterize_forward.argtypes[:-1] + [C.POINTER(RasterPlanes), vp, C.c_size_t, C.c_int, vp]
    L.psb_rasterize_backward_planes.restype = C.c_int
    L.psb_rasterize_backward_planes.argtypes = L.psb_rasterize_backward.argtypes[:-1] + [
        C.POINTER(RasterPlaneGrads), fp, vp, C.c_size_t, vp, C.c_size_t, C.c_int, C.c_int, vp]
    L.psb_mark_visible.restype = C.c_int
    L.psb_mark_visible.argtypes = [C.c_int, fp, fp, fp, u8p, vp]
    L.psb_debug_export.restype = C.c_int
    L.psb_debug_export.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp] + [vp] * 11 + [vp]
    L.psb_debug_render_bwd_occupancy.restype = C.c_int
    L.psb_debug_render_bwd_occupancy.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.psb_debug_sort_pairs.restype = C.c_int
    L.psb_debug_sort_pairs.argtypes = [vp, vp, C.c_size_t, C.c_int, vp]
    _lib = L
    return L


def check(rc, what):
    if rc < 0:
        raise PsbError(f"{what} failed ({rc}): {lib().psb_last_error().decode()}")
    return rc


def exported_symbols():
    """Names declared in include/psb200.h (used by the CPU test that checks the library exports them all)."""
    import re
    hdr = os.path.join(os.path.dirname(_HERE), "include", "psb200.h")
    txt = open(hdr).read()
    return sorted(set(re.findall(r"\b(psb_[a-z0-9_]+)\s*\(", txt)) - {"psb_alloc_fn"})
