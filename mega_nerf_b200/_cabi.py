"""ctypes binding of libmn_b200.so (the C ABI declared in include/mn_b200.h).

There is no CPU fallback: importing the package works anywhere (so that the build check and the
host-side logic can run without a GPU), but every compute entry point raises if the shared library or
a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Dict, Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libmn_b200.so')

MN_OK, MN_ERR_INVALID, MN_ERR_CUDA, MN_ERR_SHAPE, MN_ERR_SPHERE, MN_ERR_WORKSPACE, MN_ERR_UNSUPPORTED = range(7)
PREC_FP32, PREC_TC_F16, PREC_TC_F16X3 = 0, 1, 2
PRECISIONS = {'fp32': PREC_FP32, 'tc_f16': PREC_TC_F16, 'tc_f16x3': PREC_TC_F16X3}

MN_MAX_LAYERS = 16


class ModelDesc(C.Structure):
    _fields_ = [('kind', C.c_int), ('n_sub', C.c_int),
                ('pos_xyz_dim', C.c_int), ('pos_dir_dim', C.c_int), ('layers', C.c_int), ('layer_dim', C.c_int),
                ('appearance_dim', C.c_int), ('affine_appearance', C.c_int), ('appearance_count', C.c_int),
                ('rgb_dim', C.c_int), ('xyz_dim', C.c_int), ('shifted_softplus', C.c_int),
                ('n_skip', C.c_int), ('skip_layers', C.c_int * 8),
                ('boundary_margin', C.c_float), ('xyz_real', C.c_int), ('cluster_dim_start', C.c_int)]


class NerfWeights(C.Structure):
    _fields_ = [('xyz_w', C.c_void_p * MN_MAX_LAYERS), ('xyz_b', C.c_void_p * MN_MAX_LAYERS),
                ('sigma_w', C.c_void_p), ('sigma_b', C.c_void_p), ('final_w', C.c_void_p), ('final_b', C.c_void_p),
                ('dir_a_w', C.c_void_p), ('dir_a_b', C.c_void_p), ('rgb_w', C.c_void_p), ('rgb_b', C.c_void_p),
                ('embedding_a', C.c_void_p), ('affine_w', C.c_void_p), ('affine_b', C.c_void_p)]


class Rows(C.Structure):
    _fields_ = [('mode', C.c_int), ('x_d', C.c_void_p), ('cols', C.c_int), ('dirs_d', C.c_void_p),
                ('dir_stride', C.c_int64), ('idx_d', C.c_void_p), ('samples_per_ray', C.c_int)]


class Occupancy(C.Structure):
    """mn_occupancy: a reso^3 bit grid on the device and the octree frame it lives in."""
    _fields_ = [('bits', C.c_void_p), ('reso', C.c_int), ('offset', C.c_float * 3), ('scale', C.c_float * 3)]


class RenderOutputs(C.Structure):
    """mn_render_outputs: device pointers (or None) named after render_rays' result keys."""
    _fields_ = [(k, C.c_void_p) for k in ('rgb', 'depth', 'depth_var', 'bg_lambda', 'fg_rgb', 'bg_rgb', 'fg_depth', 'bg_depth',
                                          'rgb_coarse', 'bg_lambda_coarse', 'fg_rgb_coarse', 'bg_rgb_coarse')]


# name -> (restype, argtypes); every symbol of include/mn_b200.h
_P, _I, _L, _F, _Z = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
SIGNATURES = {
    'mn_abi_version': (_I, []),
    'mn_create': (_I, [C.POINTER(_P), _I]),
    'mn_destroy': (None, [_P]),
    'mn_last_error': (C.c_char_p, [_P]),
    'mn_check_status': (_I, [_P, _P]),
    'mn_launch_count': (C.c_longlong, [_P]),
    'mn_profile_enable': (_I, [_P, _I]),
    'mn_profile_read': (_I, [_P, C.POINTER(C.c_double), C.POINTER(C.c_longlong)]),
    'mn_ray_directions': (_I, [_P, _I, _I, _F, _F, _F, _F, _I, _P, _P]),
    'mn_rays': (_I, [_P, _P, _I, _P, _I, _L, _F, _F, _I, _F, _F, _P, _P]),
    'mn_rays_pairs': (_I, [_P, _P, _L, _P, _I, _P, _P, _L, _F, _F, _I, _F, _F, _P, _P]),
    'mn_gather_batch': (_I, [_P, _P, _L, _L, _P, _I, _P, _P, _I, _P, _P, _I, _P, _P]),
    'mn_debug_tp_program': (_I, [_P, _P, _I, _P]),
    'mn_debug_tp_program_mode': (_I, [_P, _I, _P, _I, _P]),
    'mn_sample_coarse': (_I, [_P, _P, _P, _P, _P, _F, _L, _I, _P, _P, _P]),
    'mn_stratify': (_I, [_P, _P, _L, _P, _F, _L, _I, _P, _P]),
    'mn_points_from_z': (_I, [_P, _P, _P, _L, _I, _P, _P]),
    'mn_sample_pdf': (_I, [_P, _P, _P, _L, _P, _P, _L, _L, _I, _I, _P, _P, _P, _P]),
    'mn_sort_cat': (_I, [_P, _P, _I, _P, _I, _L, _I, _P, _P]),
    'mn_composite': (_I, [_P, _P, _P, _P, _I, _P, _P, _P, _I, _P, _L, _I, _P, _P, _P, _P, _P, _P]),
    'mn_intersect_sphere': (_I, [_P, _P, _P, _P, _L, _P, _P]),
    'mn_points_outside': (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _P, _P, _P]),
    'mn_sh_to_rgb': (_I, [_P, _I, _P, _L, _P, _L, _I, _L, _I, _P, _P]),
    'mn_embed': (_I, [_P, _P, _L, _I, _I, _P, _P]),
    'mn_model_create': (_I, [_P, C.POINTER(ModelDesc), C.POINTER(_P)]),
    'mn_model_destroy': (None, [_P]),
    'mn_model_set_centroids': (_I, [_P, _P, _P]),
    'mn_model_set_weights': (_I, [_P, _I, C.POINTER(NerfWeights), _P]),
    'mn_model_bind_weights': (_I, [_P, _I, C.POINTER(NerfWeights)]),
    'mn_model_repack': (_I, [_P, _P, _P]),
    'mn_model_set_max_multiplicity': (_I, [_P, _I]),
    'mn_model_workspace_bytes': (_Z, [_P, _L, _I]),
    'mn_model_forward': (_I, [_P, _P, C.POINTER(Rows), _L, _I, _I, _P, _I, _P, _P, _Z, _P]),
    'mn_model_route': (_I, [_P, _P, C.POINTER(Rows), _L, _P, _P, _P]),
    'mn_model_last_stats': (_I, [_P, _P, C.POINTER(_L), C.POINTER(_L), _P]),
    'mn_model_ep_segment_rows': (_L, [_P, _L]),
    'mn_model_ep_dispatch_workspace_bytes': (_Z, [_P, _L, _I]),
    'mn_model_ep_dispatch': (_I, [_P, _P, _P, _L, _L, _I, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'mn_model_forward_assigned_workspace_bytes': (_Z, [_P, _L, _I]),
    'mn_model_forward_assigned': (_I, [_P, _P, _P, _L, _I, _I, _I, _P, _P, _Z, _P]),
    'mn_model_ep_combine': (_I, [_P, _P, _L, _P, _P, _P, _P, _P]),
    'mn_model_ep_combine_backward': (_I, [_P, _P, _L, _P, _P, _P, _P, _P]),
    'mn_model_assigned_tape_bytes': (_Z, [_P, _L, _I]),
    'mn_model_forward_assigned_train_workspace_bytes': (_Z, [_P, _L]),
    'mn_model_forward_assigned_train': (_I, [_P, _P, _P, _L, _I, _I, _L, _I, _P, _P, _Z, _P, _Z, _P]),
    'mn_model_backward_assigned_workspace_bytes': (_Z, [_P, _L, _I]),
    'mn_model_backward_assigned': (_I, [_P, _P, _L, _L, _I, _P, _P, _Z, _P, _P, _Z, _P]),
    'mn_model_density_grid_workspace_bytes': (_Z, [_P, _I]),
    'mn_model_density_grid': (_I, [_P, _P, _I, C.POINTER(_F), C.POINTER(_F), _I, _L, _L, _I, _P, _P, _Z, _P]),
    'mn_render_rays_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays': (_I, [_P, _P, _P, _P, _L, _P, _I, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _Z, _P]),
    'mn_render_rays_bg_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_bg': (_I, [_P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _P, _P, _I, _P, _P, _I, _I, _I, _I,
                               C.POINTER(RenderOutputs), _P, _Z, _P]),
    'mn_render_rays_occ_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_occ': (_I, [_P, _P, _P, _P, _L, _P, _I, _P, _I, _I, _I, _I, C.POINTER(Occupancy), _P, _P, _P, _P, _P, _P, _Z,
                                _P]),
    'mn_render_rays_bg_occ_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_bg_occ': (_I, [_P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _P, _P, _I, _P, _P, _I, _I, _I, _I,
                                   C.POINTER(Occupancy), _P, C.POINTER(RenderOutputs), _P, _Z, _P]),
    'mn_peer_gather_store': (_I, [_P, _P, _P, _L, _L, C.POINTER(C.c_void_p), _I, _P]),
    'mn_cluster_min_dist_ratios': (_I, [_P, _P, _L, _P, _I, _P, _I, _I, _F, _P, _P, _P]),
    # training (SURVEY.md §8f-1)
    'mn_composite_backward': (_I, [_P, _P, _P, _I, _P, _P, _I, _P, _L, _I, _P, _P, _P, _P, _P]),
    'mn_sh_to_rgb_backward': (_I, [_P, _I, _P, _L, _P, _L, _I, _L, _I, _P, _P, _P]),
    'mn_model_tape_bytes': (_Z, [_P, _L]),
    'mn_model_forward_train': (_I, [_P, _P, C.POINTER(Rows), _L, _I, _P, _P, _P, _Z, _P, _Z, _P]),
    'mn_model_backward_workspace_bytes': (_Z, [_P, _L]),
    'mn_model_grad_floats': (_L, [_P]),
    'mn_model_param_offsets': (_I, [_P, C.POINTER(_L), _I]),
    'mn_model_backward': (_I, [_P, _P, _L, _I, _P, _P, _Z, _P, _P, _Z, _P]),
    'mn_model_train_tc_supported': (_I, [_P]),
    'mn_model_tape_bytes_tc': (_Z, [_P, _L]),
    'mn_model_forward_train_tc': (_I, [_P, _P, C.POINTER(Rows), _L, _I, _P, _P, _P, _Z, _P, _Z, _P]),
    'mn_model_backward_workspace_bytes_tc': (_Z, [_P, _L]),
    'mn_model_backward_tc': (_I, [_P, _P, _L, _I, _P, _P, _Z, _P, _P, _Z, _P]),
    'mn_render_rays_train_tape_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train': (_I, [_P, _P, _P, _P, _L, _P, _P, _F, _I, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _Z, _P, _Z,
                                  _P]),
    'mn_render_rays_train_backward_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_backward': (_I, [_P, _P, _L, _I, _I, _I, _I, _I, _P, _P, _P, _Z, _P, _P, _Z, _P]),
    'mn_render_rays_train_bg_tape_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg': (_I, [_P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _P, _P, _P, _P, _F, _I, _P, _P, _P, _P, _P, _P, _I, _I,
                                     _I, _I, _I, _I, C.POINTER(RenderOutputs), _P, _Z, _P, _Z, _P]),
    'mn_render_rays_train_bg_backward_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg_backward': (_I, [_P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _P, _P, _P, _Z, _P, _P, _P, _Z, _P]),
    'mn_render_rays_train_occ_tape_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_occ_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_occ': (_I, [_P, _P, _P, _P, _L, _P, _P, _F, _I, _P, _P, _P, _I, _I, _I, _I, C.POINTER(Occupancy), _P, _P,
                                      _P, _P, _P, _P, _Z, _P, _Z, _P]),
    'mn_render_rays_train_occ_backward_workspace_bytes': (_Z, [_P, _L, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_occ_backward': (_I, [_P, _P, _L, _I, _I, _I, _I, _I, _P, _P, _P, _Z, _P, _P, _Z, _P]),
    'mn_render_rays_train_bg_occ_tape_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg_occ_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg_occ': (_I, [_P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _P, _P, _P, _P, _F, _I, _P, _P, _P, _P, _P, _P, _I,
                                         _I, _I, _I, _I, C.POINTER(Occupancy), _P, _I, C.POINTER(RenderOutputs), _P, _Z, _P, _Z, _P]),
    'mn_render_rays_train_bg_occ_backward_workspace_bytes': (_Z, [_P, _P, _L, _I, _I, _I, _I, _I, _I]),
    'mn_render_rays_train_bg_occ_backward': (_I, [_P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _P, _P, _P, _Z, _P, _P, _P, _Z, _P]),
    'mn_occupancy_pack': (_I, [_P, _P, _L, _F, _P, _P]),
    'mn_debug_tc_train_layout': (_I, [_P, _L, C.POINTER(_L), _I]),
    'mn_debug_tc_forward_record': (_I, [_P, _P, C.POINTER(Rows), _L, _I, _P, _P, _P, _Z, _P, _Z, _P]),
    'mn_debug_fp32_train_layout': (_I, [_P, _L, C.POINTER(_L), _I]),
    'mn_debug_weight_images': (_Z, [_P, _I, _P, _Z, _P]),
}
MN_PARAM_OFFSETS = 44
# entries of mn_debug_tc_train_layout (MN_TCL_* in include/mn_b200.h), then 2 per record image from TCL['IMG'] on
TCL = {k: i for i, k in enumerate((
    'ENGINE', 'N_TILES', 'TAPE_BYTES', 'TAPE_COUNTERS', 'TAPE_SLOT_ROW', 'TAPE_SLOT_W', 'TAPE_XREG', 'TAPE_ACT', 'TAPE_F32',
    'X_TILE', 'ACT_TILE', 'KPE', 'KAUX', 'HC', 'GC', 'F32_SIGMA', 'F32_RGB', 'F32_ID', 'F32_ROWS', 'G32_SIGMA', 'G32_RGB',
    'G32_ROWS', 'BWD_BYTES', 'BWD_DZ', 'BWD_GF32', 'BWD_EMB', 'BWD_SCALE', 'BWD_EMB_K', 'BWD_HEAD_TILES', 'BWD_DZG',
    'BWD_PP0', 'BWD_PP1', 'N_IMG', 'TRAIN', 'IMG'))}
# entries of mn_debug_fp32_train_layout (MN_F32L_* in include/mn_b200.h)
F32L = {k: i for i, k in enumerate((
    'TM', 'N_TILES', 'CHUNK_TILES', 'TAPE_BYTES', 'TAPE_COUNTERS', 'TAPE_SLOT_ROW', 'TAPE_SLOT_W', 'TAPE_ACT', 'BWD_BYTES',
    'BWD_GRAD', 'A_PE', 'A_AUX', 'A_H', 'A_F', 'A_G', 'A_RGB', 'A_LIN', 'A_SIG', 'A_ID', 'A_TOTAL', 'G_Z', 'G_FINAL', 'G_DIRA',
    'G_RGB', 'G_SIG', 'G_TOTAL', 'COUNT'))}

_lib = None
_lock = threading.Lock()
_ctx: Dict[int, int] = {}


def load_library():
    """dlopen the in-tree library and bind every symbol (no GPU needed for this step)."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f'{LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                                   f'(or `python mega_nerf_b200/build.py`). There is no CPU fallback.')
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)      # AttributeError = symbol missing: fail loudly
                fn.restype = res
                fn.argtypes = args
            if lib.mn_abi_version() != 1:
                raise RuntimeError('libmn_b200.so ABI version mismatch')
            _lib = lib
    return _lib


def lib():
    return load_library()


def ctx(device: torch.device) -> int:
    """Per-device native context."""
    if device.type != 'cuda':
        raise RuntimeError('mega_nerf_b200 runs on CUDA (sm_90a) tensors only; there is no CPU path')
    idx = device.index if device.index is not None else torch.cuda.current_device()
    with _lock:
        h = _ctx.get(idx)
    if h is None:
        L = lib()
        out = C.c_void_p()
        rc = L.mn_create(C.byref(out), idx)
        if rc != MN_OK:
            msg = L.mn_last_error(out).decode() if out.value else 'mn_create failed'
            raise RuntimeError(f'libmn_b200: {msg}')
        with _lock:
            _ctx[idx] = out.value
        h = out.value
    return h


def check(rc: int, h: int):
    if rc == MN_OK:
        return
    msg = lib().mn_last_error(h).decode()
    if rc in (MN_ERR_SHAPE, MN_ERR_SPHERE):
        raise Exception(msg)          # the reference raises plain Exception with this text
    raise RuntimeError(f'libmn_b200 error {rc}: {msg}')


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def stream_of(device: torch.device):
    return torch.cuda.current_stream(device).cuda_stream


def f32c(t: torch.Tensor) -> torch.Tensor:
    """Contiguous fp32 view/copy of a CUDA tensor."""
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()
