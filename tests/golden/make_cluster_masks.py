"""Generate tests/golden/cluster_masks_v1.pt by running the UNMODIFIED reference script
scripts/create_cluster_masks.py (main(), CPU) on a tiny synthetic dataset directory written to a temp dir.
Needs a checkout of the reference:    MEGA_NERF_REFERENCE=<path> python tests/golden/make_cluster_masks.py
Pins oracle/mn_oracle.py::image_cluster_masks / cluster_min_dist_ratios (SURVEY.md §8f-3)."""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile
import types
from argparse import Namespace
from pathlib import Path
from zipfile import ZipFile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402

C, O = MG.C, MG.O

# scripts/create_cluster_masks.py imports mega_nerf.opts (needs configargparse, absent here); main() never calls it
stub = types.ModuleType('mega_nerf.opts')
stub.get_opts_base = lambda: None
sys.modules['mega_nerf.opts'] = stub
spec = importlib.util.spec_from_file_location('ref_create_cluster_masks', os.path.join(MG.REF, 'scripts', 'create_cluster_masks.py'))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)


def main():
    case = C.cluster_mask_case()
    with tempfile.TemporaryDirectory() as tmp:
        ds = Path(tmp) / 'dataset'
        for sub in ('train', 'val'):
            (ds / sub / 'metadata').mkdir(parents=True)
        torch.save({'origin_drb': torch.zeros(3), 'pose_scale_factor': 1.0}, ds / 'coordinates.pt')
        for i, im in enumerate(case['images']):
            sub = 'val' if i == len(case['images']) - 1 else 'train'
            torch.save({'c2w': im['c2w'], 'intrinsics': im['intrinsics'], 'W': im['W'], 'H': im['H']},
                       ds / sub / 'metadata' / f'{i:06d}.pt')
        out = Path(tmp) / 'masks'
        hp = Namespace(dataset_path=str(ds), output=str(out), segmentation_path=None, grid_dim=case['grid_dim'],
                       ray_samples=case['ray_samples'], ray_chunk_size=case['ray_chunk_size'], dist_chunk_size=64 * 1024 * 1024,
                       resume=False, ray_altitude_range=case['ray_altitude_range'], near=case['near'], far=case['far'],
                       cluster_2d=case['cluster_2d'], boundary_margin=case['boundary_margin'], center_pixels=case['center_pixels'])
        ref.main(hp)
        params = torch.load(out / 'params.pt', map_location='cpu', weights_only=False)
        K = params['centroids'].shape[0]
        masks = []
        for i in range(len(case['images'])):
            name = f'{i:06d}.pt'
            per = []
            for k in range(K):
                with ZipFile(out / str(k) / name) as zf:
                    with zf.open(name) as f:
                        per.append(torch.load(f, map_location='cpu'))
            masks.append(torch.stack(per))
    # the oracle agrees
    cams = torch.stack([im['c2w'][:3, 3] for im in case['images']])
    cent, mn, mx = O.grid_centroids_from_cameras(cams, case['grid_dim'])
    assert torch.equal(cent, params['centroids']), (cent, params['centroids'])
    zs = torch.linspace(0, 1, case['ray_samples'])
    bad = 0
    for im, m in zip(case['images'], masks):
        got = O.image_cluster_masks(im['W'], im['H'], im['intrinsics'], im['c2w'], params['near'], params['far'],
                                    params['ray_altitude_range'], case['center_pixels'], zs, cent, case['cluster_2d'],
                                    case['boundary_margin'], case['ray_chunk_size'])
        bad += int((got != m).sum())
        print(f'image {im["W"]}x{im["H"]}: pixels per cluster {[int(x.sum()) for x in m]}')
    assert bad == 0, f'oracle != reference on {bad} mask bits'
    torch.save({'masks': masks, 'centroids': params['centroids'], 'near': params['near'], 'far': params['far'],
                'ray_altitude_range': [float(x) for x in params['ray_altitude_range']]}, C.CLUSTER_GOLDEN_PATH)
    print(f'wrote {C.CLUSTER_GOLDEN_PATH} ({os.path.getsize(C.CLUSTER_GOLDEN_PATH) / 1e3:.1f} kB); oracle == reference')


if __name__ == '__main__':
    main()
