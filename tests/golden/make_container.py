"""Generate tests/golden/container_v1.pt: a merged TorchScript container exactly as the reference's
scripts/merge_submodules.py:70-77 writes it (MegaNeRFContainer of reference NeRF sub-modules, scripted),
with small seeded networks.  Needs a checkout of the reference:
    MEGA_NERF_REFERENCE=<path> python tests/golden/make_container.py
The fixture is the on-disk INPUT format of the path (SURVEY.md §8f-4); loading it needs no reference code."""
from __future__ import annotations

import os
import sys

import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402

C, O = MG.C, MG.O
from mega_nerf.models.mega_nerf_container import MegaNeRFContainer  # noqa: E402


def main():
    fg, bg, cents = C.container_nets()
    subs = [MG.ref_nerf(fg.spec, w) for w in fg.weights]
    bsubs = [MG.ref_nerf(bg.spec, w) for w in bg.weights]
    cont = MegaNeRFContainer(subs, bsubs, cents, torch.IntTensor([1, 2, 2]), torch.tensor([-1.0, -1.0, -1.0]),
                             torch.tensor([1.0, 1.0, 1.0]), fg.spec.pos_dir_dim > 0, fg.spec.appearance_dim > 0, True)
    torch.jit.save(torch.jit.script(cont.eval()), C.CONTAINER_PATH)
    back = torch.jit.load(C.CONTAINER_PATH, map_location='cpu')
    assert len(back.centroids) == 4 and back.cluster_2d is True
    C.split_golden_bytes(C.CONTAINER_PATH)          # committed as byte parts below 1 MB each (C.container_path() joins them)
    print(f'wrote {C.CONTAINER_PATH}.part*')


if __name__ == '__main__':
    main()
