"""Alias this package over the reference's module names so that the reference's own
train.py / eval.py / Runner import this package's path unchanged:

    import mega_nerf_b200; mega_nerf_b200.install()
    from mega_nerf.runner import Runner        # picks up render_rays / get_nerf / get_rays from here

Replaced names (runner.py:33-35, filesystem_dataset.py:18):
    mega_nerf.rendering.render_rays, mega_nerf.models.model_utils.get_nerf / get_bg_nerf,
    mega_nerf.ray_utils.get_rays / get_ray_directions / get_rays_batch, the model classes, and
    FilesystemDataset._load_chunk_inner (the chunk loader's ray generation, filesystem_dataset.py:95-131), and
    mega_nerf.runner.DataLoader (training batches gathered on the device, runner.py:23, 228-236).
"""
from __future__ import annotations

import importlib
import sys
import types


def install(patch_loaded: bool = True) -> None:
    from . import modules, raygen, render, sh

    def mod(name, **attrs):
        m = sys.modules.get(name)
        if m is None:
            try:
                m = importlib.import_module(name)       # keep whatever else the reference module defines
            except Exception:
                m = types.ModuleType(name)
                sys.modules[name] = m
                parent, _, leaf = name.rpartition('.')
                if parent and parent in sys.modules:
                    setattr(sys.modules[parent], leaf, m)
        for k, v in attrs.items():
            setattr(m, k, v)
        return m

    if 'mega_nerf' not in sys.modules:
        try:
            importlib.import_module('mega_nerf')
        except Exception:
            pkg = types.ModuleType('mega_nerf')
            pkg.__path__ = []
            sys.modules['mega_nerf'] = pkg
    if 'mega_nerf.models' not in sys.modules:
        try:
            importlib.import_module('mega_nerf.models')
        except Exception:
            sub = types.ModuleType('mega_nerf.models')
            sub.__path__ = []
            sys.modules['mega_nerf.models'] = sub
            sys.modules['mega_nerf'].models = sub

    mod('mega_nerf.rendering', render_rays=render.render_rays)
    mod('mega_nerf.ray_utils', get_ray_directions=raygen.get_ray_directions, get_rays=raygen.get_rays,
        get_rays_batch=raygen.get_rays_batch)
    mod('mega_nerf.spherical_harmonics', eval_sh=sh.eval_sh)
    mod('mega_nerf.models.nerf', NeRF=modules.NeRF, Embedding=modules.Embedding, ShiftedSoftplus=modules.ShiftedSoftplus)
    mod('mega_nerf.models.mega_nerf', MegaNeRF=modules.MegaNeRF)
    mod('mega_nerf.models.cascade', Cascade=modules.Cascade)
    mod('mega_nerf.models.model_utils', get_nerf=modules.get_nerf, get_bg_nerf=modules.get_bg_nerf)
    if patch_loaded:
        # modules that did `from mega_nerf.rendering import render_rays` before install()
        for name, target in (('mega_nerf.runner', {'render_rays': render.render_rays, 'get_nerf': modules.get_nerf,
                                                   'get_bg_nerf': modules.get_bg_nerf, 'get_rays': raygen.get_rays,
                                                   'get_ray_directions': raygen.get_ray_directions}),
                             ('mega_nerf.datasets.filesystem_dataset', {'get_rays_batch': raygen.get_rays_batch})):
            m = sys.modules.get(name)
            if m is not None:
                for k, v in target.items():
                    if hasattr(m, k):
                        setattr(m, k, v)
    patch_loader()
    patch_data_loader()


def patch_data_loader() -> bool:
    """Bind the device batches (mega_nerf_b200/batches.py) over the `DataLoader` name `Runner.train()` builds its loaders with
    (runner.py:23, 228-236) if `mega_nerf.runner` is - or can be - imported.  torch's own DataLoader is not touched."""
    from . import batches
    m = sys.modules.get('mega_nerf.runner')
    if m is None:
        try:
            m = importlib.import_module('mega_nerf.runner')
        except Exception:       # no reference on the path, or its imports (cv2, lpips, ...) unavailable
            return False
    m.DataLoader = batches.data_loader
    return True


def patch_loader() -> bool:
    """Bind the fused chunk loader (mega_nerf_b200/loader.py, SURVEY.md §8f-6) over
    `FilesystemDataset._load_chunk_inner` (filesystem_dataset.py:95-131) if that module is - or can be - imported."""
    from . import loader
    m = sys.modules.get('mega_nerf.datasets.filesystem_dataset')
    if m is None:
        try:
            m = importlib.import_module('mega_nerf.datasets.filesystem_dataset')
        except Exception:       # e.g. no reference on the path, or its imports (np.int, pyarrow) unavailable
            return False
    cls = getattr(m, 'FilesystemDataset', None)
    if cls is None:
        return False
    if getattr(cls._load_chunk_inner, '__module__', '') != loader.__name__:
        cls._reference_load_chunk_inner = cls._load_chunk_inner
        cls._load_chunk_inner = loader._load_chunk_inner
    return True
