"""GPU: the fused cluster-mask kernel (mn_cluster_min_dist_ratios, SURVEY.md §8f-3) against the oracle and the
reference's own masks.

Every float op of the reference is restated with its own rounding (the accumulators of cdist's matmul path are
bit-identical to an in-order FMA chain), but torch's vectorised CPU `sqrt` is not correctly rounded: it is 1 ulp off
IEEE `sqrtf` on ~0.6 % of inputs (measured on the CPU: 6141 of 1e6 random inputs; numpy's and CUDA's
agree with the correctly rounded value everywhere).  So the distance ratios may differ from the CPU oracle by an ulp
or two and are compared to 4 ulp; the boolean masks - the actual output - must be identical wherever the ratio is not
within 1e-6 of the margin, and identical everywhere on the committed reference fixture."""
import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M

pytestmark = pytest.mark.gpu


def test_min_dist_ratios():
    from mega_nerf_b200 import cluster_masks as CM
    for (ny, nz), c2d, S in (((2, 4), True, 1000), ((5, 5), True, 257), ((2, 4), False, 64), ((6, 8), True, 100)):
        rays = O.synthetic_rays(300, seed=ny * 10 + nz, far=1.2)
        cent = O.grid_centroids(ny, nz)
        if not c2d:
            cent = cent.clone()
            cent[:, 0] = torch.rand(cent.shape[0], generator=torch.Generator().manual_seed(1)) * 0.4 - 0.2
        zs = torch.linspace(0, 1, S)
        want = O.cluster_min_dist_ratios(rays, zs, cent, c2d)
        got, mask = CM.min_dist_ratios(rays.to(DEV), zs.to(DEV), cent.to(DEV), c2d, 1.15)
        rel = ((got.cpu() - want).abs() / want).max()
        assert float(rel) <= 4 * 2.0 ** -24, float(rel)
        decided = ((want - 1.15).abs() > 1e-6 * 1.15).t()
        assert torch.equal(mask.cpu().bool()[decided], (want <= 1.15).t()[decided])
        assert torch.equal(mask.cpu().bool(), (got.cpu() <= 1.15).t())          # mask and ratio outputs agree with each other


def test_image_masks_match_reference_script():
    from mega_nerf_b200 import cluster_masks as CM
    gd = torch.load(C.CLUSTER_GOLDEN_PATH, map_location='cpu', weights_only=False)
    case = C.cluster_mask_case()
    zs = torch.linspace(0, 1, case['ray_samples'])
    wrong = total = 0
    for im, want in zip(case['images'], gd['masks']):
        got = CM.image_cluster_masks(im['W'], im['H'], im['intrinsics'], im['c2w'], gd['near'], gd['far'],
                                     gd['ray_altitude_range'], case['center_pixels'], zs, gd['centroids'], case['cluster_2d'],
                                     case['boundary_margin'], DEV)
        assert got.shape == want.shape and got.dtype == torch.bool
        wrong += int((got.cpu() != want).sum())
        total += want.numel()
    # ray generation on the GPU is within 5e-7 of the oracle, not bit-exact (tests/test_gpu_parity.py::test_raygen), so a
    # pixel whose ratio sits within an ulp of the margin may flip; none does on this fixture
    assert wrong == 0, f'{wrong} of {total} mask bits differ'
