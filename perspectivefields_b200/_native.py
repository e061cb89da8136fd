"""ctypes binding of libpf_b200.so (C ABI declared in include/pf_b200.h) and its in-tree build recipe.

There is no CPU fallback: importing this module works without a GPU (so the ABI can be inspected), but every
compute entry point needs the CUDA library and an H100 (sm_90a).
"""
import ctypes
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_HERE, "libpf_b200.so")
SRC_DIR = os.path.join(_HERE, "csrc")
OBJ_DIR = os.path.join(_HERE, "build")
HEADER = os.path.join(ROOT, "include", "pf_b200.h")

PF_F32, PF_BF16 = 0, 1
PF_PARAM_NONE, PF_PARAM_CENTERED, PF_PARAM_UNCENTERED = 0, 1, 2

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
LINK_FLAGS = ["-shared", "-ldl"]


class pf_model_desc(ctypes.Structure):
    _fields_ = [("gravity_classes", ctypes.c_int), ("latitude_classes", ctypes.c_int), ("param_net", ctypes.c_int),
                ("param_input_size", ctypes.c_int), ("pixel_mean", ctypes.c_float * 3), ("pixel_std", ctypes.c_float * 3)]


class pf_camera(ctypes.Structure):
    """include/pf_b200.h: struct pf_camera."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("focal_rel", ctypes.c_double), ("elevation", ctypes.c_double),
                ("roll", ctypes.c_double), ("cx_rel", ctypes.c_double), ("cy_rel", ctypes.c_double),
                ("up_offset", ctypes.c_int64), ("lat_offset", ctypes.c_int64)]


class pf_pano_view(ctypes.Structure):
    """include/pf_b200.h: struct pf_pano_view (one view of pf_pano_views)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("f", ctypes.c_double), ("xi", ctypes.c_double),
                ("az", ctypes.c_double), ("el", ctypes.c_double), ("roll", ctypes.c_double),
                ("im_offset", ctypes.c_int64), ("field_offset", ctypes.c_int64)]


class pf_equi_view(ctypes.Structure):
    """include/pf_b200.h: struct pf_equi_view (one view of pf_equi_views)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("vfov", ctypes.c_double), ("azimuth", ctypes.c_double),
                ("elevation", ctypes.c_double), ("roll", ctypes.c_double), ("ar", ctypes.c_double), ("offset", ctypes.c_int64)]


class pf_field_image(ctypes.Structure):
    """include/pf_b200.h: struct pf_field_image (one image of pf_field_errors)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("pred_up_offset", ctypes.c_int64), ("pred_up_stride", ctypes.c_int64 * 3),
                ("pred_lat_offset", ctypes.c_int64), ("gt_up_offset", ctypes.c_int64), ("gt_up_stride", ctypes.c_int64 * 3),
                ("gt_lat_offset", ctypes.c_int64), ("mask_offset", ctypes.c_int64)]


class pf_fit_image(ctypes.Structure):
    """include/pf_b200.h: struct pf_fit_image (one image of pf_fit_camera)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("up_offset", ctypes.c_int64), ("up_stride", ctypes.c_int64 * 3),
                ("lat_offset", ctypes.c_int64), ("mask_offset", ctypes.c_int64), ("init", ctypes.c_double * 5)]


class pf_rectify_image(ctypes.Structure):
    """include/pf_b200.h: struct pf_rectify_image (one image of pf_rectify_views)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("out_height", ctypes.c_int32), ("out_width", ctypes.c_int32),
                ("in_offset", ctypes.c_int64), ("out_offset", ctypes.c_int64), ("mask_offset", ctypes.c_int64), ("map_offset", ctypes.c_int64)]


class pf_pano_crop(ctypes.Structure):
    """include/pf_b200.h: struct pf_pano_crop (the crop of one view of pf_fit_panorama)."""
    _fields_ = [("vfov", ctypes.c_double), ("azimuth", ctypes.c_double), ("elevation", ctypes.c_double), ("roll", ctypes.c_double),
                ("ar", ctypes.c_double)]


class pf_rotate_pano(ctypes.Structure):
    """include/pf_b200.h: struct pf_rotate_pano (one panorama of pf_rotate_panoramas)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("in_offset", ctypes.c_int64), ("out_offset", ctypes.c_int64),
                ("map_offset", ctypes.c_int64)]


PF_RECTIFY_SAME, PF_RECTIFY_VFOV, PF_RECTIFY_FILL, PF_RECTIFY_FILL_COMMON = 0, 1, 2, 4
PF_RECTIFY_BILINEAR, PF_RECTIFY_NEAREST = 0, 1

PF_EQUI_U8, PF_EQUI_F32 = 0, 1
PF_EQUI_BILINEAR, PF_EQUI_NEAREST = 0, 1
PF_EQUI_CAST, PF_EQUI_UNIT = 0, 1


class pf_draw_canvas(ctypes.Structure):
    """include/pf_b200.h: struct pf_draw_canvas (one canvas of pf_draw_fields)."""
    _fields_ = [("height", ctypes.c_int32), ("width", ctypes.c_int32), ("img_offset", ctypes.c_int64), ("out_offset", ctypes.c_int64),
                ("lat_offset", ctypes.c_int64), ("up_offset", ctypes.c_int64), ("up_stride", ctypes.c_int64 * 3),
                ("density", ctypes.c_int32), ("arrow_inv_len", ctypes.c_int32), ("arrow_rgb", ctypes.c_float * 3),
                ("alpha_fill", ctypes.c_float), ("alpha_line", ctypes.c_float), ("draw_lat", ctypes.c_int32), ("draw_up", ctypes.c_int32)]


class pf_batch(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int),
                ("images_u8", ctypes.c_void_p), ("image_offset", ctypes.POINTER(ctypes.c_int64)),
                ("images_chw", ctypes.c_void_p),
                ("height", ctypes.POINTER(ctypes.c_int32)), ("width", ctypes.POINTER(ctypes.c_int32)),
                ("pred_gravity", ctypes.c_void_p), ("pred_latitude", ctypes.c_void_p),
                ("gravity_original", ctypes.c_void_p), ("gravity_original_offset", ctypes.POINTER(ctypes.c_int64)),
                ("latitude_original", ctypes.c_void_p), ("latitude_original_offset", ctypes.POINTER(ctypes.c_int64)),
                ("params", ctypes.c_void_p)]


class pf_confidence(ctypes.Structure):
    """include/pf_b200.h: struct pf_confidence (the head-confidence outputs of pf_forward_confidence)."""
    _fields_ = [("gravity", ctypes.c_void_p), ("latitude", ctypes.c_void_p), ("gravity_original", ctypes.c_void_p),
                ("latitude_original", ctypes.c_void_p)]


class pf_tma_pred(ctypes.Structure):
    """include/pf_b200.h: struct pf_tma_pred (fused prediction tail of one group)."""
    _fields_ = [("w", ctypes.c_void_p), ("b", ctypes.c_void_p), ("out", ctypes.c_void_p), ("nc", ctypes.c_int), ("mode", ctypes.c_int)]


def _fields(spec):
    """"int a, b; ptr c; i64 d" -> ctypes fields in that order (ptr: any pointer, i64: int64_t)."""
    types = {"int": ctypes.c_int, "ptr": ctypes.c_void_p, "i64": ctypes.c_int64}
    out = []
    for decl in spec.split(";"):
        t, names = decl.split(None, 1)
        out += [(n.strip(), types[t]) for n in names.split(",")]
    return out


class pf_tma_op(ctypes.Structure):
    """include/pf_b200.h: struct pf_tma_op (one launch of the TMA -> wgmma engine, pf_op_tma)."""
    _fields_ = _fields("int mode; i64 M; int K, B, H, W, Cin, N, groups; ptr a_hi, a_lo; int lda, a_c0, a_gc; ptr a2_hi, a2_lo;"
                       "int lda2, c_split, a2_c0; ptr w_hi, w_lo, bias; int bias_mode, bias_gstride, act; ptr gamma, res;"
                       "int ldr, r_coff, r_gcoff, res_relu; ptr res2; int ldr2, r2_coff, r2_gcoff; ptr C; int ldc, c_coff, c_gcoff;"
                       "ptr s_hi, s_lo; int lds, s_coff, s_gcoff, split_relu, phase4, npred") + \
        [("pred", pf_tma_pred * 2)] + _fields("int force_bn, force_kb, picked_bn, picked_kb, force_sched, picked_sched")


def _sources():
    return sorted(os.path.join(SRC_DIR, f) for f in os.listdir(SRC_DIR) if f.endswith((".cu", ".cuh", ".h"))) + [HEADER]


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(s) > t for s in _sources())


def _stale(obj):
    """An object is stale when it, or the dependency list nvcc wrote beside it, is missing or older than a file it was built from."""
    if not (os.path.exists(obj) and os.path.exists(obj + ".d")):
        return True
    deps = open(obj + ".d").read().replace("\\\n", " ").split(":", 1)[1].split()
    t = os.path.getmtime(obj)
    return any(not os.path.exists(d) or os.path.getmtime(d) > t for d in deps)


def _nvcc(args, out, verbose):
    cmd = [os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + args + ["-o", out + ".tmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    os.replace(out + ".tmp", out)
    if verbose:
        print(r.stderr)


def build(force=False, verbose=False):
    """Compile every csrc/*.cu for sm_90a (nvcc cross-compiles without a GPU), in parallel, into build/, and link them into
    libpf_b200.so next to this file.  Objects whose sources have not changed since they were built are reused unless force."""
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    objs = {os.path.join(OBJ_DIR, f[:-3] + ".o"): os.path.join(SRC_DIR, f) for f in sorted(os.listdir(SRC_DIR)) if f.endswith(".cu")}
    flags = NVCC_FLAGS + (["-Xptxas=-v"] if verbose else [])
    with ThreadPoolExecutor(os.cpu_count()) as pool:
        list(pool.map(lambda o: _nvcc(flags + ["-MD", "-MF", o + ".d", "-c", objs[o]], o, verbose), [o for o in objs if force or _stale(o)]))
    _nvcc(LINK_FLAGS + list(objs), LIB_PATH, verbose)
    return LIB_PATH


_lib = None


def lib():
    """Load libpf_b200.so (raises if it has not been built: the product has no other compute path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(perspectivefields_b200 has no CPU or PyTorch fallback)")
    # PF_B200_LIB: an alternative build of the SAME library (A/B timing of kernel changes on one box: tools/ab.sh)
    L = ctypes.CDLL(os.environ.get("PF_B200_LIB") or LIB_PATH)
    vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    sig = {
        "pf_abi_version": (i32, []),
        "pf_last_error": (ctypes.c_char_p, []),
        "pf_kernel_launch_count": (i64, []),
        "pf_resize_table_stats": (i32, [vp, ctypes.POINTER(i64), ctypes.POINTER(i64)]),
        "pf_create": (i32, [i32, ctypes.POINTER(pf_model_desc), ctypes.POINTER(vp)]),
        "pf_create_sized": (i32, [i32, ctypes.POINTER(pf_model_desc), i32, i32, ctypes.POINTER(vp)]),
        "pf_destroy": (i32, [vp]),
        "pf_set_weight": (i32, [vp, ctypes.c_char_p, vp, i64, i32]),
        "pf_finalize": (i32, [vp]),
        "pf_workspace_bytes": (i64, [vp, i32, i32]),
        "pf_forward": (i32, [vp, ctypes.POINTER(pf_batch), vp, i64, vp]),
        "pf_forward_confidence": (i32, [vp, ctypes.POINTER(pf_batch), ctypes.POINTER(pf_confidence), vp, i64, vp]),
        "pf_param_workspace_bytes": (i64, [vp, i32]),
        "pf_param_forward": (i32, [vp, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_param_train_workspace_bytes": (i64, [vp, i32]),
        "pf_param_train_forward": (i32, [vp, i32, vp, vp, vp, vp, i64, vp]),
        "pf_param_backward": (i32, [vp, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_param_grad_numel": (i64, []),
        "pf_param_grad_entry": (i32, [i32, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(i64), ctypes.POINTER(i64)]),
        "pf_profile_enable": (i32, [vp, i32]),
        "pf_profile_read": (i32, [vp, ctypes.POINTER(ctypes.c_double)]),
        "pf_profile_kernels_enable": (i32, [vp, i32]),
        "pf_profile_kernels_read": (i32, [vp, ctypes.c_char_p, i32]),
        "pf_debug_enable": (i32, [vp, i32]),
        "pf_debug_count": (i32, [vp]),
        "pf_debug_name": (ctypes.c_char_p, [vp, i32]),
        "pf_debug_numel": (i64, [vp, ctypes.c_char_p]),
        "pf_debug_copy": (i32, [vp, ctypes.c_char_p, vp, i64, vp]),
        "pf_op_conv_gemm": (i32, [vp, i32, i32, i32, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp, vp]),
        "pf_op_tma": (i32, [ctypes.POINTER(pf_tma_op), vp]),
        "pf_op_tma_bf16": (i32, [ctypes.POINTER(pf_tma_op), vp]),
        "pf_op_conv1_ring": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "pf_tma_pick_tile": (i32, [i32, i64, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32)]),
        "pf_set_option": (i32, [vp, ctypes.c_char_p, i32]),
        "pf_camera_fields": (i32, [i32, ctypes.POINTER(pf_camera), i32, vp, vp, vp]),
        "pf_camera_fields_vp": (i32, [i32, ctypes.POINTER(pf_camera), ctypes.POINTER(ctypes.c_double), i32, vp, vp, vp]),
        "pf_draw_fields": (i32, [i32, ctypes.POINTER(pf_draw_canvas), i32, vp, vp, vp, vp, vp]),
        "pf_pano_views": (i32, [i32, vp, i32, i32, ctypes.POINTER(pf_pano_view), i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "pf_equi_views": (i32, [i32, vp, i32, i32, i32, i32, ctypes.POINTER(pf_equi_view), i32, i32, i32, i32, vp, vp]),
        "pf_encode_fields": (i32, [i32, i32, i32, i32, vp, ctypes.POINTER(i64), vp, ctypes.POINTER(i64), i32, i32, i32, vp, vp, vp]),
        "pf_head_losses_workspace": (i64, [i32, i32, i32, i32, i32]),
        "pf_head_losses": (i32, [i32, i32, i32, i32, i32, vp, vp, i32, vp, vp, i32, i32, f32, f32, vp, vp, i64, vp]),
        "pf_field_errors_workspace": (i64, [ctypes.POINTER(pf_field_image), i32, i32]),
        "pf_field_errors": (i32, [i32, ctypes.POINTER(pf_field_image), i32, vp, vp, vp, vp, vp, i32, ctypes.POINTER(ctypes.c_double), i32,
                                  vp, vp, vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_camera_workspace": (i64, [ctypes.POINTER(pf_fit_image), i32]),
        "pf_fit_camera": (i32, [i32, ctypes.POINTER(pf_fit_image), i32, vp, vp, vp, i32, ctypes.c_double, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_camera_groups_workspace": (i64, [ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32]),
        "pf_fit_camera_groups": (i32, [i32, ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32, vp, vp, vp, i32, ctypes.c_double,
                                       i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_camera_weighted": (i32, [i32, ctypes.POINTER(pf_fit_image), i32, vp, vp, vp, vp, ctypes.POINTER(i64), ctypes.POINTER(i64), i32,
                                         ctypes.c_double, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_camera_groups_weighted": (i32, [i32, ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32, vp, vp, vp, vp,
                                                ctypes.POINTER(i64), ctypes.POINTER(i64), i32, ctypes.c_double, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_camera_sequences_workspace": (i64, [ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32]),
        "pf_fit_camera_sequences": (i32, [i32, ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32, vp, vp, vp, vp,
                                          ctypes.POINTER(i64), ctypes.POINTER(i64), i32, ctypes.c_double, i32, ctypes.c_double, ctypes.c_double,
                                          vp, vp, vp, vp, vp, i64, vp]),
        "pf_fit_panorama_workspace": (i64, [ctypes.POINTER(pf_fit_image), i32, ctypes.POINTER(ctypes.c_int32), i32]),
        "pf_fit_panorama": (i32, [i32, ctypes.POINTER(pf_fit_image), ctypes.POINTER(pf_pano_crop), i32, ctypes.POINTER(ctypes.c_int32), i32, vp,
                                  vp, vp, vp, ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.POINTER(ctypes.c_double), ctypes.c_double, i32,
                                  vp, vp, vp, vp, vp, vp, vp, i64, vp]),
        "pf_rotate_panoramas_workspace": (i64, [ctypes.POINTER(pf_rotate_pano), i32]),
        "pf_rotate_panoramas": (i32, [i32, ctypes.POINTER(pf_rotate_pano), i32, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp]),
        "pf_rectify_workspace": (i64, [ctypes.POINTER(pf_rectify_image), i32]),
        "pf_rectify_views": (i32, [i32, ctypes.POINTER(pf_rectify_image), i32, vp, vp, vp, vp, i32, vp, i32, i32, ctypes.c_double, i32,
                                   ctypes.POINTER(ctypes.c_int32), vp, vp, vp, i64, vp]),
        "pf_op_pn_wgrad": (i32, [vp, i32, vp, vp, vp, i32, i32, i64, i32, i32, vp, ctypes.POINTER(i32), ctypes.POINTER(i32), vp]),
        "pf_op_pn_colsum": (i32, [vp, i64, i32, vp, vp]),
        "pf_op_pn_ln_bwd": (i32, [vp, vp, i64, i32, vp, vp, vp, vp]),
        "pf_op_pn_dw7_bwd": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp, ctypes.POINTER(i32), vp]),
        "pf_op_pn_stem_bwd": (i32, [vp, vp, vp, i32, i32, i32, vp, vp, ctypes.POINTER(i32), vp]),
        "pf_op_pn_fields_grad": (i32, [vp, i32, i32, i32, i32, i32, vp, vp, vp]),
        "pf_op_pn_tail_bwd": (i32, [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]),
        "pf_op_pn_pw2_grads": (i32, [vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
        "pf_op_pn_gelu_bwd": (i32, [vp, vp, i64, vp, vp, vp]),
        "pf_op_pn_scale_split": (i32, [vp, vp, i64, i32, vp, vp, vp]),
        "pf_op_pn_col2im2": (i32, [vp, i32, i32, i32, i32, vp, vp]),
        "pf_op_layernorm": (i32, [vp, vp, i64, i32, vp, vp, f32, vp]),
        "pf_op_attention_tc": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_attention_tc_bf16": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_attention_tc_keys": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
        "pf_op_dwconv3x3_gelu": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp]),
        "pf_op_dwconv7x7": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp]),
        "pf_op_upsample2x": (i32, [vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_layernorm_ex": (i32, [vp, vp, vp, vp, vp, vp, i64, i32, vp, vp, f32, i32, i32, i32, vp]),
        "pf_op_dwconv3x3_gelu_ex": (i32, [vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
        "pf_op_upsample2x_ex": (i32, [vp, i32, i32, vp, i32, i32, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_stem_gather": (i32, [vp, i32, i32, i32, i32, vp, vp, vp]),
        "pf_op_pn_stem": (i32, [vp, i32, i32, i32, vp, vp, vp, vp]),
        "pf_op_pack_fields": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, vp]),
        "pf_op_param_tail": (i32, [vp, i32, i32, vp, vp, vp, vp, i32, vp, vp, vp]),
        "pf_op_pred_tail": (i32, [vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_preprocess": (i32, [vp, i32, i32, ctypes.POINTER(f32), ctypes.POINTER(f32), vp, vp]),
        "pf_op_preprocess_sized": (i32, [vp, i32, i32, i32, i32, ctypes.POINTER(f32), ctypes.POINTER(f32), vp, vp]),
        "pf_op_resize_u8": (i32, [vp, i32, i32, i32, i32, vp, vp]),
        "pf_op_resize_f32": (i32, [vp, i32, i32, i32, i32, i32, vp, vp]),
        "pf_op_argmax_decode": (i32, [vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_fill_stream": (i32, [vp, i64, f32, vp]),
        "pf_op_pred_argmax_decode": (i32, [vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_subbin_decode": (i32, [vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_pred_subbin_decode": (i32, [vp, i32, i32, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
        "pf_op_flip_merge_reg": (i32, [vp, vp, vp, vp, i32, i32, i32, vp]),
        "pf_op_flip_pred": (i32, [vp, i32, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]),
        "pf_op_postprocess": (i32, [vp, vp, i32, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32), vp, ctypes.POINTER(i64), vp,
                                    ctypes.POINTER(i64), i32, vp]),
        "pf_op_postprocess_sized": (i32, [vp, vp, i32, i32, i32, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32), vp,
                                          ctypes.POINTER(i64), vp, ctypes.POINTER(i64), i32, vp]),
        "pf_comm_unique_id": (i32, [vp]),
        "pf_comm_create": (i32, [i32, i32, i32, vp, ctypes.POINTER(vp)]),
        "pf_comm_destroy": (i32, [vp]),
        "pf_gather": (i32, [vp, i32, i32, ctypes.POINTER(vp), ctypes.POINTER(i64), ctypes.POINTER(ctypes.c_int32), vp]),
        "pf_jpeg_create": (i32, [i32, i32, ctypes.POINTER(vp)]),
        "pf_jpeg_destroy": (i32, [vp]),
        "pf_jpeg_info": (i32, [vp, vp, i64, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32)]),
        "pf_jpeg_decode_batch": (i32, [vp, i32, ctypes.POINTER(vp), ctypes.POINTER(i64), ctypes.POINTER(ctypes.c_int32),
                                       ctypes.POINTER(ctypes.c_int32), vp, ctypes.POINTER(i64), vp]),
    }
    for name, (res, args) in sig.items():
        try:
            fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
        except AttributeError:
            if os.environ.get("PF_B200_LIB"):   # an older build under A/B test may predate an entry point
                continue
            raise
        fn.restype, fn.argtypes = res, args
    if L.pf_abi_version() != 3:
        raise RuntimeError("libpf_b200.so ABI version mismatch")
    _lib = L
    return L


EXPORTS = ["pf_abi_version", "pf_last_error", "pf_kernel_launch_count", "pf_resize_table_stats", "pf_create", "pf_create_sized", "pf_destroy", "pf_set_weight",
           "pf_finalize", "pf_workspace_bytes", "pf_forward", "pf_forward_confidence", "pf_param_workspace_bytes", "pf_param_forward", "pf_param_train_workspace_bytes",
           "pf_param_train_forward", "pf_param_backward", "pf_param_grad_numel", "pf_param_grad_entry", "pf_profile_enable", "pf_profile_read", "pf_profile_kernels_enable",
           "pf_profile_kernels_read", "pf_set_option", "pf_debug_enable", "pf_debug_count", "pf_debug_name", "pf_debug_numel",
           "pf_debug_copy", "pf_camera_fields", "pf_camera_fields_vp", "pf_pano_views", "pf_equi_views", "pf_draw_fields",
           "pf_encode_fields", "pf_head_losses_workspace", "pf_head_losses", "pf_field_errors_workspace", "pf_field_errors",
           "pf_fit_camera_workspace", "pf_fit_camera", "pf_fit_camera_groups_workspace", "pf_fit_camera_groups",
           "pf_fit_camera_weighted", "pf_fit_camera_groups_weighted", "pf_fit_camera_sequences_workspace", "pf_fit_camera_sequences",
           "pf_fit_panorama_workspace", "pf_fit_panorama",
           "pf_rotate_panoramas_workspace", "pf_rotate_panoramas",
           "pf_rectify_workspace", "pf_rectify_views", "pf_comm_unique_id", "pf_comm_create", "pf_comm_destroy", "pf_gather",
           "pf_jpeg_create", "pf_jpeg_destroy", "pf_jpeg_info", "pf_jpeg_decode_batch",
           "pf_op_conv_gemm", "pf_op_tma", "pf_op_tma_bf16", "pf_op_conv1_ring", "pf_tma_pick_tile", "pf_op_layernorm",
           "pf_op_attention_tc", "pf_op_attention_tc_bf16", "pf_op_attention_tc_keys", "pf_op_dwconv3x3_gelu",
           "pf_op_dwconv7x7", "pf_op_upsample2x", "pf_op_preprocess", "pf_op_preprocess_sized", "pf_op_fill_stream", "pf_op_resize_u8",
           "pf_op_resize_f32", "pf_op_argmax_decode", "pf_op_pred_argmax_decode", "pf_op_subbin_decode", "pf_op_pred_subbin_decode",
           "pf_op_flip_merge_reg", "pf_op_flip_pred", "pf_op_postprocess", "pf_op_postprocess_sized",
           "pf_op_pn_wgrad", "pf_op_pn_colsum", "pf_op_pn_ln_bwd", "pf_op_pn_dw7_bwd", "pf_op_pn_stem_bwd", "pf_op_pn_fields_grad",
           "pf_op_pn_tail_bwd", "pf_op_pn_pw2_grads", "pf_op_pn_gelu_bwd", "pf_op_pn_scale_split", "pf_op_pn_col2im2",
           "pf_op_layernorm_ex", "pf_op_dwconv3x3_gelu_ex", "pf_op_upsample2x_ex", "pf_op_stem_gather", "pf_op_pn_stem",
           "pf_op_pack_fields", "pf_op_param_tail", "pf_op_pred_tail"]


class PfError(RuntimeError):
    pass


def check(status):
    if status < 0:
        raise PfError(f"libpf_b200: {lib().pf_last_error().decode()} (status {status})")
    return status
