"""ctypes loader for libfluid_b200.so (the C ABI of include/fluid.h).

No fallback of any kind: if the shared library is missing this raises; if there is no sm_90 GPU
fluid_create() fails with FLUID_ERR_NO_DEVICE and FluidError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
# FLUID_B200_SO: load another build of the same library (tuning experiments: register caps etc.)
SO_PATH = os.environ.get("FLUID_B200_SO") or os.path.join(_HERE, "libfluid_b200.so")
CSRC = os.path.join(_HERE, "csrc")

# every symbol include/fluid.h declares (tests check the .so exports exactly these)
SYMBOLS = [
    "fluid_abi_version", "fluid_config_default", "fluid_get_resolution", "fluid_create",
    "fluid_create_slab", "fluid_nccl_unique_id", "fluid_p2p_export", "fluid_p2p_connect", "fluid_p2p_disable", "fluid_destroy", "fluid_resize", "fluid_step",
    "fluid_splat", "fluid_splats", "fluid_set_param", "fluid_set_param_f64", "fluid_get_param", "fluid_stat", "fluid_pass_curl", "fluid_pass_vorticity",
    "fluid_pass_divergence", "fluid_pass_clear_pressure", "fluid_pass_jacobi",
    "fluid_pass_pressure_solve", "fluid_pass_gradient_subtract", "fluid_pass_advect_velocity",
    "fluid_pass_advect_dye", "fluid_pass_curl_vorticity_divergence", "fluid_field_elems",
    "fluid_field_dims", "fluid_read", "fluid_write", "fluid_read_device", "fluid_write_device", "fluid_pressure_solve_host", "fluid_render", "fluid_render_band", "fluid_render_postfx", "fluid_render_keywords", "fluid_capture", "fluid_capture_device", "fluid_render_canvas", "fluid_sync",
    "fluid_timing_last", "fluid_host_alloc", "fluid_host_free", "fluid_mark", "fluid_elapsed_ms", "fluid_launch_count", "fluid_device_ptr",
    "fluid_last_error", "fluid_create_batch", "fluid_members", "fluid_splats_batch", "fluid_render_canvas_batch",
    "fluid_capture_batch", "fluid_set_param_members", "fluid_get_param_members", "fluid_step_members",
    "fluid_splats_device", "fluid_splats_batch_device", "fluid_read_members", "fluid_write_members",
    "fluid_reset_members", "fluid_render_canvas_members", "fluid_capture_members", "fluid_render_canvas_looks",
    "fluid_capture_looks",
]

FLUID_OK = 0
ERR_NAMES = {-1: "FLUID_ERR_INVALID", -2: "FLUID_ERR_NO_DEVICE", -3: "FLUID_ERR_CUDA",
             -4: "FLUID_ERR_NCCL", -5: "FLUID_ERR_HALO", -6: "FLUID_ERR_NOMEM"}

FIELD = {"velocity": 0, "dye": 1, "pressure": 2, "divergence": 3, "curl": 4}
PARAM = {"DENSITY_DISSIPATION": 0, "VELOCITY_DISSIPATION": 1, "PRESSURE": 2,
         "PRESSURE_ITERATIONS": 3, "CURL": 4, "SPLAT_RADIUS": 5, "ASPECT": 6, "JACOBI_BLOCK": 7, "BACKGROUND": 8}
FLAG_UNFUSED, FLAG_NO_GRAPH, FLAG_NAIVE_JACOBI, FLAG_TILED_PASSES, FLAG_HALF_STORAGE = 0x1, 0x2, 0x4, 0x8, 0x10
FLAG_HALF_POSTFX = 0x20         # fp16 bloom / sunrays targets like the reference's FBOs (include/fluid.h)
FLAG_NEAREST_FILTERING = 0x40   # NEAREST display / post-FX / resize samplers, the reference without float linear filtering
FLAG_LINEAR_ADVECTION = 0x80    # advection through LINEAR samplers, the reference with float linear filtering
# display keywords of render() (updateKeywords, S:1160-1166): FLUID_DISPLAY_* of include/fluid.h
DISPLAY_SHADING, DISPLAY_BLOOM, DISPLAY_SUNRAYS = 0x1, 0x2, 0x4
STAT = {"launches": 0, "jacobi_launches": 1, "halo_launches": 2, "halo_exchanges": 3,
        "graph_captures": 4, "graph_launches": 5, "halo_transport_p2p": 6, "cvd_stream_launches": 7,
        "gradient_stream_launches": 8, "jacobi_exact_streams": 9, "advect4_launches": 10, "gathers": 11}


class FluidError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("sim_w", C.c_int32), ("sim_h", C.c_int32), ("dye_w", C.c_int32), ("dye_h", C.c_int32),
                ("density_dissipation", C.c_float), ("velocity_dissipation", C.c_float),
                ("pressure", C.c_float), ("pressure_iterations", C.c_int32), ("curl", C.c_float),
                ("splat_radius", C.c_float), ("aspect", C.c_float), ("device", C.c_int32),
                ("flags", C.c_uint32), ("jacobi_block", C.c_int32)]


class PostFX(C.Structure):
    _fields_ = [("bloom_iterations", C.c_int32), ("bloom_resolution", C.c_int32), ("bloom_intensity", C.c_double),
                ("bloom_threshold", C.c_double), ("bloom_soft_knee", C.c_double), ("sunrays_resolution", C.c_int32),
                ("sunrays_weight", C.c_double)]


class Look(C.Structure):
    """fluid_look: one image's post-FX sliders and background in fluid_render_canvas_looks / fluid_capture_looks."""
    _fields_ = [("bloom_intensity", C.c_double), ("bloom_threshold", C.c_double), ("bloom_soft_knee", C.c_double),
                ("sunrays_weight", C.c_double), ("back_r", C.c_float), ("back_g", C.c_float), ("back_b", C.c_float),
                ("transparent", C.c_int32)]


class Timing(C.Structure):
    _fields_ = [("curl_vort_div_ms", C.c_float), ("jacobi_ms", C.c_float), ("gradient_ms", C.c_float),
                ("advect_velocity_ms", C.c_float), ("advect_dye_ms", C.c_float), ("total_ms", C.c_float),
                ("jacobi_launches", C.c_int32), ("total_launches", C.c_int32)]


def build(force: bool = False) -> str:
    """Compile libfluid_b200.so in-tree with nvcc for sm_90a (works without a GPU)."""
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")) or f == "Makefile"]
    srcs.append(os.path.join(os.path.dirname(_HERE), "include", "fluid.h"))
    stale = (not os.path.exists(SO_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(SO_PATH) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", CSRC, "-s"], stdout=subprocess.DEVNULL)
    return SO_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise FileNotFoundError(
            f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU or PyTorch fallback for this library)")
    L = C.CDLL(SO_PATH)
    vp, i, f, fp, sz = C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_float), C.c_size_t
    L.fluid_abi_version.restype = i
    L.fluid_config_default.argtypes = [C.POINTER(Config)]; L.fluid_config_default.restype = None
    L.fluid_get_resolution.argtypes = [i, i, i, C.POINTER(i), C.POINTER(i)]; L.fluid_get_resolution.restype = None
    L.fluid_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.fluid_create_batch.argtypes = [C.POINTER(Config), i, C.POINTER(vp)]
    L.fluid_members.argtypes = [vp]
    L.fluid_create_slab.argtypes = [C.POINTER(Config), i, i, vp, sz, C.POINTER(vp)]
    L.fluid_nccl_unique_id.argtypes = [vp, sz]
    L.fluid_p2p_export.argtypes = [vp, vp, sz]
    L.fluid_p2p_connect.argtypes = [vp, vp, vp]
    L.fluid_p2p_disable.argtypes = [vp]
    L.fluid_destroy.argtypes = [vp]; L.fluid_destroy.restype = None
    L.fluid_resize.argtypes = [vp, i, i, i, i]
    L.fluid_step.argtypes = [vp, f]
    L.fluid_splat.argtypes = [vp] + [f] * 7
    L.fluid_splats.argtypes = [vp, fp, i]
    L.fluid_splats_batch.argtypes = [vp, C.POINTER(C.c_int32), fp, i]
    L.fluid_splats_device.argtypes = [vp, vp, i]
    L.fluid_splats_batch_device.argtypes = [vp, vp, vp, i]
    L.fluid_set_param.argtypes = [vp, i, f]
    L.fluid_set_param_f64.argtypes = [vp, i, C.c_double]
    L.fluid_get_param.argtypes = [vp, i, fp]
    L.fluid_set_param_members.argtypes = [vp, i, C.POINTER(C.c_double), i]
    L.fluid_get_param_members.argtypes = [vp, i, fp, i]
    L.fluid_step_members.argtypes = [vp, fp, i]
    L.fluid_stat.argtypes = [vp, i]; L.fluid_stat.restype = C.c_uint64
    for n in ("curl", "divergence", "clear_pressure", "pressure_solve", "gradient_subtract"):
        getattr(L, "fluid_pass_" + n).argtypes = [vp]
    for n in ("vorticity", "advect_velocity", "advect_dye", "curl_vorticity_divergence"):
        getattr(L, "fluid_pass_" + n).argtypes = [vp, f]
    L.fluid_pass_jacobi.argtypes = [vp, i]
    L.fluid_field_elems.argtypes = [vp, i]; L.fluid_field_elems.restype = sz
    L.fluid_field_dims.argtypes = [vp, i] + [C.POINTER(i)] * 4
    L.fluid_read.argtypes = [vp, i, vp, sz]
    L.fluid_write.argtypes = [vp, i, vp, sz]
    L.fluid_read_device.argtypes = [vp, i, vp, sz]
    L.fluid_write_device.argtypes = [vp, i, vp, sz]
    L.fluid_pressure_solve_host.argtypes = [vp, vp, vp, i]
    L.fluid_render.argtypes = [vp, i, i, i, f, f, f, vp, sz]
    L.fluid_render_band.argtypes = [vp, i, C.POINTER(i), C.POINTER(i)]
    L.fluid_render_postfx.argtypes = [vp, i, i, C.POINTER(PostFX), vp, i, i, f, f, f, vp, sz, vp, vp]
    L.fluid_render_keywords.argtypes = [vp, i, i, C.c_uint32, C.POINTER(PostFX), vp, i, i, f, f, f, vp, sz, vp, vp]
    L.fluid_capture.argtypes = [vp, i, i, i, i, C.c_uint32, i, C.POINTER(PostFX), vp, i, i, f, f, f, vp, sz]
    L.fluid_capture_device.argtypes = L.fluid_capture.argtypes
    L.fluid_render_canvas.argtypes = [vp, i, i, C.c_uint32, i, C.POINTER(PostFX), vp, i, i, f, f, f, vp, sz, i]
    L.fluid_render_canvas_batch.argtypes = L.fluid_render_canvas.argtypes
    L.fluid_capture_batch.argtypes = L.fluid_capture.argtypes + [i]
    ip = C.POINTER(C.c_int32)
    L.fluid_read_members.argtypes = [vp, i, ip, i, vp, sz, i]
    L.fluid_write_members.argtypes = [vp, i, ip, i, vp, sz, i]
    L.fluid_reset_members.argtypes = [vp, ip, i]
    L.fluid_render_canvas_members.argtypes = L.fluid_render_canvas_batch.argtypes + [ip, i]
    L.fluid_capture_members.argtypes = L.fluid_capture_batch.argtypes + [ip, i]
    lk = C.POINTER(Look)
    L.fluid_render_canvas_looks.argtypes = [vp, i, i, C.c_uint32, C.POINTER(PostFX), vp, i, i, lk, vp, sz, i, ip, i]
    L.fluid_capture_looks.argtypes = [vp, i, i, i, i, C.c_uint32, C.POINTER(PostFX), vp, i, i, lk, vp, sz, i, ip, i]
    L.fluid_sync.argtypes = [vp]
    L.fluid_host_alloc.argtypes = [sz]; L.fluid_host_alloc.restype = vp
    L.fluid_host_free.argtypes = [vp]; L.fluid_host_free.restype = None
    L.fluid_timing_last.argtypes = [vp, C.POINTER(Timing)]
    L.fluid_mark.argtypes = [vp, i]
    L.fluid_elapsed_ms.argtypes = [vp, fp]
    L.fluid_launch_count.argtypes = [vp]; L.fluid_launch_count.restype = C.c_uint64
    L.fluid_device_ptr.argtypes = [vp, i]; L.fluid_device_ptr.restype = vp
    L.fluid_last_error.argtypes = [vp]; L.fluid_last_error.restype = C.c_char_p
    _lib = L
    return L
