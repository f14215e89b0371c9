"""ctypes binding of libovg.so (include/ovg.h).  There is NO fallback: if the shared library is missing or the
device is not an H100 (sm_90) the import / first call fails loudly."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OVG_LIB_PATH") or os.path.join(_HERE, "libovg.so")   # override: A/B kernel builds

EPI_BF16, EPI_RESID, EPI_QKV, EPI_HEADTAIL = 0, 1, 2, 3
ROWS_IDENT, ROWS_DENSE2PAD, ROWS_PAD, ROWS_PIXSHUF = 0, 1, 2, 3
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2

_vp, _i, _ll, _f = C.c_void_p, C.c_int, C.c_longlong, C.c_float


class GemmArgs(C.Structure):
    """Mirror of ``ovg_gemm_args`` (include/ovg.h); field order must match exactly."""
    _fields_ = [
        ("a", _vp), ("a_rows", _ll), ("a_cols", _i), ("lda", _ll),
        ("b", _vp), ("n", _i), ("ldb", _ll),
        ("m", _i),
        ("num_taps", _i), ("tap_off", _i * 9),
        ("epi", _i),
        ("bias", _vp), ("act", _i), ("out", _vp), ("ldo", _ll),
        ("table", _vp), ("table_rows", _i),
        ("skip1", _vp), ("skip2", _vp),
        ("rowmap", _i), ("gh", _i), ("gw", _i), ("ps", _i), ("cout", _i),
        ("gamma", _vp), ("row_index", _vp),
        ("q_out", _vp), ("k_out", _vp), ("v_out", _vp),
        ("C", _i), ("ntok", _i), ("T", _i), ("nspecial", _i), ("wp", _i), ("maxpos", _i),
        ("qn_w", _vp), ("qn_b", _vp), ("kn_w", _vp), ("kn_b", _vp),
        ("rope_cos", _vp), ("rope_sin", _vp), ("qscale", _f),
        ("w2", _vp), ("b2", _vp), ("outc", _i), ("head_act", _i), ("preds", _vp), ("conf", _vp),
        ("block_n", _i), ("qk_norm", _i), ("rope", _i),
        ("k_peers", _vp * 8), ("v_peers", _vp * 8), ("n_peers", _i), ("peer_ntok", _i), ("peer_tok_off", _ll),
        ("f16", _i),
    ]


class BlockWeights(C.Structure):
    """Mirror of ``ovg_block_weights``."""
    _fields_ = [(n, _vp) for n in ("ln1_w", "ln1_b", "w_qkv", "b_qkv", "qn_w", "qn_b", "kn_w", "kn_b", "w_proj", "b_proj", "g1",
                                   "ln2_w", "ln2_b", "w_fc1", "b_fc1", "w_fc2", "b_fc2", "g2")]


class AggregatorDesc(C.Structure):
    """Mirror of ``ovg_aggregator_desc``."""
    _fields_ = [("C", _i), ("registers", _i), ("depth", _i), ("patch", _i),
                ("frame_blocks", C.POINTER(BlockWeights)), ("global_blocks", C.POINTER(BlockWeights)),
                ("cam_tok", _vp), ("reg_tok", _vp), ("placeholder", _vp), ("depth_w", _vp), ("depth_b", _vp), ("ones_c", _vp),
                ("keep_layers", _i * 4)]


class DinoDesc(C.Structure):
    """Mirror of ``ovg_dino_desc``."""
    _fields_ = [("C", _i), ("registers", _i), ("depth", _i), ("patch", _i), ("kpad", _i),
                ("blocks", C.POINTER(BlockWeights)), ("w_patch", _vp), ("b_patch", _vp), ("norm_w", _vp), ("norm_b", _vp),
                ("ones_c", _vp)]


class DptFusion(C.Structure):
    """Mirror of ``ovg_dpt_fusion``."""
    _fields_ = [("rcu1", _vp * 4), ("rcu2", _vp * 4), ("oc_w", _vp), ("oc_b", _vp)]


class DptDesc(C.Structure):
    """Mirror of ``ovg_dpt_desc``."""
    _fields_ = [("C2", _i), ("feat", _i), ("patch", _i), ("outc", _i), ("oc", _i * 4),
                ("proj_w", _vp * 4), ("proj_b", _vp * 4), ("up_w", _vp * 2), ("up_b", _vp * 2), ("down_w", _vp), ("down_b", _vp),
                ("rn_w", _vp * 4), ("fus", DptFusion * 4), ("oc1_w", _vp), ("oc1_b", _vp), ("oc2_w", _vp), ("oc2_b", _vp),
                ("w2", _vp), ("b2", _vp), ("f16", _i)]


class CameraDesc(C.Structure):
    """Mirror of ``ovg_camera_desc``."""
    _fields_ = [("D", _i), ("heads", _i), ("trunk_depth", _i), ("trunk", C.POINTER(BlockWeights)),
                ("token_norm_w", _vp), ("token_norm_b", _vp), ("trunk_norm_w", _vp), ("trunk_norm_b", _vp), ("empty_pose", _vp),
                ("embed_w", _vp), ("embed_b", _vp), ("mod_w", _vp), ("mod_b", _vp), ("fc1_w", _vp), ("fc1_b", _vp),
                ("fc2_w", _vp), ("fc2_b", _vp)]


class ContextParallelDesc(C.Structure):
    """Mirror of ``ovg_context_parallel``."""
    _fields_ = [("rank", _i), ("world", _i), ("views_total", _i), ("k_peers", (_vp * 8) * 2), ("v_peers", (_vp * 8) * 2),
                ("flag_peers", _vp * 8), ("epoch_counter", _vp), ("cam_peers", _vp * 8)]


_pp = C.POINTER(_vp)
EXPORTS = {
    "ovg_version": (C.c_int, []),
    "ovg_last_error": (C.c_char_p, []),
    "ovg_device_check": (C.c_int, []),
    "ovg_launch_count": (C.c_longlong, []),
    "ovg_gemm": (C.c_int, [C.POINTER(GemmArgs), _vp]),
    "ovg_attention": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp]),
    "ovg_attention_scratch_bytes": (C.c_longlong, []),
    "ovg_peer_barrier": (C.c_int, [C.POINTER(_vp), _vp, _i, _i, _vp]),
    "ovg_layernorm": (C.c_int, [_vp, _i, _ll, _vp, _i, _ll, _i, _i, _vp, _vp, _f, _i, _i, _i, _vp]),
    "ovg_image_im2col": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "ovg_assemble_tokens": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "ovg_inject_snapshot": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "ovg_depth_im2col": (C.c_int, [_vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "ovg_im2col3x3s2": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "ovg_dpt_tail_supported": (C.c_int, [_i, _i, _i, _i, _i]),
    "ovg_dpt_tail_scratch_bytes": (C.c_longlong, [_i, _i]),
    "ovg_dpt_tail": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "ovg_upsample_bilinear": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "ovg_preprocess_image": (C.c_int, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "ovg_preprocess_image_canvas": (C.c_int, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i,
                                              _i, _i, _f, _vp]),
    "ovg_preprocess_depth": (C.c_int, [_vp, _ll, _ll, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp]),
    "ovg_prepare_cameras": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "ovg_pose_decode": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "ovg_unproject_depth": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "ovg_conf_percentile_mask": (C.c_int, [_vp, _ll, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "ovg_point_cloud_workspace_bytes": (_ll, [_ll]),
    "ovg_point_cloud_count": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _ll, _vp, _vp]),
    "ovg_point_cloud_gather": (C.c_int, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp, _vp, _ll, _vp]),
    "ovg_point_cloud_center": (C.c_int, [_vp, _ll, _vp, _ll, _vp, _vp]),
    "ovg_point_cloud_scale": (C.c_int, [_vp, _ll, _ll, _vp, _ll, _vp, _vp]),
    "ovg_match_workspace_bytes": (_ll, [_i, _ll, _i]),
    "ovg_match_index": (C.c_int, [_vp, _vp, _i, _ll, _i, _vp, _ll, _vp]),
    "ovg_match_query": (C.c_int, [_vp, _i, _i, _ll, _vp, _ll, _vp, _vp]),
    "ovg_match_gather": (C.c_int, [_vp, _i, _i, _ll, _i, _vp, _ll, _vp, _vp, _vp]),
    "ovg_match_pair": (C.c_int, [_vp, _i, _i, _ll, _i, _vp, _ll, _vp, _vp, _vp]),
    "ovg_tracks_workspace_bytes": (_ll, [_i, _ll]),
    "ovg_tracks_assign": (C.c_int, [_vp, _vp, _i, _i, _ll, _i, _vp, _ll, _vp, _ll, _vp, _vp]),
    "ovg_tracks_gather": (C.c_int, [_vp, _vp, _vp, _i, _ll, _i, _i, _ll, _ll, _vp, _ll, _vp, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp, _vp, _vp]),
    "ovg_ba_workspace_bytes": (_ll, [_i, _ll, _ll]),
    "ovg_bundle_adjust": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _ll, _i, _i, _i, C.c_double, _vp, _ll, _vp, _vp, _vp, _vp,
                                    _vp, _vp, _vp, _vp]),
    "ovg_mesh_workspace_bytes": (_ll, [_i, _i, _i]),
    "ovg_mesh_count": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _ll, _vp, _vp]),
    "ovg_mesh_faces": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp]),
    "ovg_mesh_compact": (C.c_int, [_vp, _vp, _i, _i, _i, _vp, _ll, _vp, _vp, _vp, _vp]),
    "ovg_tsdf_workspace_bytes": (_ll, [_i, _i, _i, _i, _i, _i]),
    "ovg_tsdf_bounds": (C.c_int, [_vp, _vp, _i, _i, _i, _vp, _ll, _vp, _vp]),
    "ovg_tsdf_integrate": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _f, _f, _f, _f, _vp, _ll, _vp, _vp, _vp]),
    "ovg_tsdf_count": (C.c_int, [_vp, _i, _i, _i, _vp, _ll, _vp, _vp]),
    "ovg_tsdf_extract": (C.c_int, [_vp, _vp, _i, _i, _i, _f, _f, _f, _f, _vp, _ll, _vp, _vp, _vp, _vp]),
    "ovg_sky_workspace_bytes": (_ll, [_i, _i, _i]),
    "ovg_segment_sky": (C.c_int, [_vp, _i, _ll, _ll, _ll, _i, _i, _i, _vp, _vp, _ll, _vp, _vp, _vp]),
    "ovg_sky_mask_conf": (C.c_int, [_vp, _vp, _ll, _vp, _vp]),
    "ovg_fps_workspace_bytes": (_ll, [_i, _ll]),
    "ovg_farthest_point_sample": (C.c_int, [_vp, _i, _ll, _i, _vp, _i, _vp, _ll, _vp, _vp]),
    "ovg_ranking_workspace_bytes": (_ll, [_ll, _i]),
    "ovg_compute_ranking": (C.c_int, [_vp, _i, _ll, _ll, _ll, _ll, C.c_double, _i, _i, _ll, _vp, _ll, _vp, _vp, _vp]),
    "ovg_sim3_workspace_bytes": (_ll, [_ll]),
    "ovg_sim3_estimate": (C.c_int, [_vp, _vp, _vp, _ll, _vp, _ll, _vp, _vp, _vp]),
    "ovg_sim3_apply": (C.c_int, [_vp, _i, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ovg_jpeg_plan_create": (C.c_int, [_pp, C.POINTER(_ll), _i, _i, _pp]),
    "ovg_jpeg_plan_destroy": (None, [_vp]),
    "ovg_jpeg_plan_file": (C.c_int, [_vp, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "ovg_jpeg_plan_stream_bytes": (_ll, [_vp]),
    "ovg_jpeg_plan_workspace_bytes": (_ll, [_vp]),
    "ovg_jpeg_plan_subsequences": (_ll, [_vp]),
    "ovg_jpeg_plan_segments": (_ll, [_vp]),
    "ovg_jpeg_plan_segment": (C.c_int, [_vp, _ll, C.POINTER(_i), C.POINTER(_ll), C.POINTER(_ll), C.POINTER(_i), C.POINTER(_i)]),
    "ovg_jpeg_plan_fill_stream": (C.c_int, [_vp, _vp]),
    "ovg_jpeg_plan_rounds": (C.c_int, [_vp]),
    "ovg_jpeg_decode": (C.c_int, [_vp, _vp, _pp, _vp, _vp, _ll, _vp]),
    # ---- runtime (handle-level sequences)
    "ovg_aggregator_create": (C.c_int, [C.POINTER(AggregatorDesc), _pp]),
    "ovg_aggregator_destroy": (None, [_vp]),
    "ovg_aggregator_workspace_bytes": (_ll, [_vp, _i, _i, _i, _i, _i]),
    "ovg_aggregator_forward": (C.c_int, [_vp, C.POINTER(ContextParallelDesc), _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i,
                                         _i, _i, _i, _i, _vp, _ll, _pp, _vp, _pp, _vp]),
    "ovg_dino_create": (C.c_int, [C.POINTER(DinoDesc), _pp]),
    "ovg_dino_destroy": (None, [_vp]),
    "ovg_dino_workspace_bytes": (_ll, [_vp, _i, _i, _i]),
    "ovg_dino_forward": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _ll, _vp, _vp]),
    "ovg_dpt_create": (C.c_int, [C.POINTER(DptDesc), _pp]),
    "ovg_dpt_destroy": (None, [_vp]),
    "ovg_dpt_workspace_bytes": (_ll, [_vp, _i, _i, _i]),
    "ovg_dpt_forward": (C.c_int, [_vp, _pp, _i, _i, _i, _i, _i, _i, _i, _pp, _vp, _vp, _i, _vp, _vp, _vp, _ll, _vp]),
    "ovg_camera_create": (C.c_int, [C.POINTER(CameraDesc), _pp]),
    "ovg_camera_destroy": (None, [_vp]),
    "ovg_camera_workspace_bytes": (_ll, [_vp, _i]),
    "ovg_camera_forward": (C.c_int, [_vp, _vp, _i, _i, _i, _vp, _vp, _ll, _vp]),
    "ovg_runtime_time_attention": (None, [_i]),
    "ovg_runtime_attention_split": (None, [_i]),
    "ovg_runtime_attention_times": (C.c_int, [_vp, _i]),
}
PERCENTILE_WORKSPACE_BYTES = 6 * 8 + 512 * 4 + 4 * 4


def DEPTH_SCRATCH_DOUBLES(B: int) -> int:
    """Mirror of OVG_DEPTH_SCRATCH_DOUBLES (include/ovg.h)."""
    return B * (2 * 1024 + 1)

JPEG_DEVICE = 0                 # OVG_JPEG_DEVICE; the other OVG_JPEG_* values are host-routing reasons
JPEG_MIN_SUBSEQ_BITS = 32       # OVG_JPEG_MIN_SUBSEQ_BITS


class JpegPlan:
    """Owner of an ``ovg_jpeg_plan`` (host code, no GPU needed): routing, sizes and the staging stream of a list of files."""

    def __init__(self, files, subseq_bits: int = 0):
        l = load()
        self._lib = l
        self.n = len(files)
        files = [bytes(f) for f in files]                  # no copy for bytes; the plan copies what it keeps
        ptrs = (_vp * max(self.n, 1))(*[C.cast(C.c_char_p(f), _vp) for f in files])
        sizes = (_ll * max(self.n, 1))(*[len(f) for f in files])
        h = _vp()
        check(l.ovg_jpeg_plan_create(ptrs, sizes, self.n, int(subseq_bits), C.byref(h)))
        self.handle = h
        self.files = []
        for i in range(self.n):
            r, w, hh, c = _i(), _i(), _i(), _i()
            check(l.ovg_jpeg_plan_file(h, i, C.byref(r), C.byref(w), C.byref(hh), C.byref(c)))
            self.files.append((r.value, hh.value, w.value, c.value))       # (route, height, width, components)
        self.stream_bytes = l.ovg_jpeg_plan_stream_bytes(h)
        self.workspace_bytes = l.ovg_jpeg_plan_workspace_bytes(h)
        self.subsequences = l.ovg_jpeg_plan_subsequences(h)

    def segments(self):
        """[(file, stream byte offset, bytes, first MCU, MCUs)] in stream order."""
        out = []
        for k in range(self._lib.ovg_jpeg_plan_segments(self.handle)):
            f, o, nb, m, nm = _i(), _ll(), _ll(), _i(), _i()
            check(self._lib.ovg_jpeg_plan_segment(self.handle, k, C.byref(f), C.byref(o), C.byref(nb), C.byref(m), C.byref(nm)))
            out.append((f.value, o.value, nb.value, m.value, nm.value))
        return out

    def fill_stream(self, dst_ptr: int) -> None:
        check(self._lib.ovg_jpeg_plan_fill_stream(self.handle, dst_ptr))

    def rounds(self) -> int:
        return self._lib.ovg_jpeg_plan_rounds(self.handle)

    def __del__(self):
        if getattr(self, "handle", None):
            self._lib.ovg_jpeg_plan_destroy(self.handle)
            self.handle = None


_lib: Optional[C.CDLL] = None
_device_ok = False


class OvgError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load libovg.so and bind every symbol declared in include/ovg.h (no GPU needed for this step)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OvgError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU / PyTorch fallback for the hot path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def lib() -> C.CDLL:
    """Library handle for compute calls: additionally requires an H100 (sm_90) as the current device."""
    global _device_ok
    l = load()
    if not _device_ok:
        if not torch.cuda.is_available():
            raise OvgError("libovg needs a CUDA device (H100); torch.cuda.is_available() is False")
        torch.cuda.current_device()          # make sure the primary context exists
        check(l.ovg_device_check())
        _device_ok = True
    return l


def check(rc: int) -> None:
    if rc != 0:
        raise OvgError(f"libovg error {rc}: {load().ovg_last_error().decode()}")


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream
