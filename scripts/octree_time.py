"""Times the network queries of octree extraction: python scripts/octree_time.py [--out FILE] [--quick]

Each line runs one unmodified reference function of scripts/create_octree.py (the copy build() makes under oracle/_ref/, with the
stub svox of tests/golden/make_octree.py) on this repository's network modules, then the mega_nerf_b200.octree call that replaces
it, on the same network and box, and checks the two outputs against each other:
  step0  _auto_scale at init_grid_depth 8 (256^3 rows)                     vs octree.auto_scale
  step1  _step1's grid at 512^3 with masking_mode 'sigma'                  vs octree.grid_sigmas + occupied_points
  step2  _step2 over 10^5 cells x 256 samples                              vs octree.cell_colors (+ the copy into the tree)
for the mega-nerf shape (8 x 256 MegaNeRF, 2 x 4 centroids, margin 1.15) and, step 0 only, the nerf config's 2048-wide Cascade
fine network.  Precision tc_f16 (the module default).  Each line: ms (host clock around the call, ending in a device sync),
rows/s, algorithmic trunk TFLOP/s (trunk Linear FLOPs per row x the mean number of sub-modules a row is routed to, measured
on 2^18 rows of the box), peak device memory.  Prints the card name and power limit read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'golden')):
    sys.path.insert(0, p)
import torch  # noqa: E402
from torch import nn  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import octree as T  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
import make_octree as MO  # noqa: E402

DEV = torch.device('cuda:0')
CHUNK = 32768


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


class Recorder(nn.Module):
    """The network as the reference calls it, keeping column 0 of every sigma_only result (the reference keeps none in step 0)."""

    def __init__(self, p: nn.Module):
        super().__init__()
        self.p, self.kept = p, []

    def forward(self, *args, **kw):
        out = self.p(*args, **kw)
        if kw.get('sigma_only'):
            self.kept.append(out[:, 0])
        return out


def trunk_flops_per_row(spec: O.NerfSpec) -> int:
    L, f = spec.layer_dim, 0
    for i in range(spec.layers):
        f += 2 * L * (spec.in_xyz if i == 0 else (spec.in_xyz + L if i in spec.skip_layers else L))
    return f


def multiplicity(net: O.Net, offset, scale) -> float:
    if net.kind != 'mega':
        return 1.0
    g = torch.Generator().manual_seed(0)
    x = ((torch.rand(1 << 18, 3, generator=g) - offset) / scale)
    _, w = O.route(net, x)
    return float((w > 0).sum(1).float().mean()) if w is not None else 1.0


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t) * 1e3, torch.cuda.max_memory_allocated() / 2 ** 30


def line(step, shape, who, ms, rows, flops_row, mult, mem, **extra):
    out = dict(step=step, net=shape, impl=who, ms=round(ms, 2), rows=rows, rows_per_s=rows / ms * 1e3,
               trunk_tflops=rows * flops_row * mult / ms / 1e9, mult=round(mult, 3), peak_mem_gib=round(mem, 3), **extra)
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--quick', action='store_true', help='smaller sizes (a rehearsal, not a measurement)')
    args = ap.parse_args()
    print(f'card: {smi("name,power.limit,clocks.max.sm")}', flush=True)
    ref = MO.load_reference()
    assert ref is not None, 'oracle/_ref/ is missing: run build() where the reference source tree is available'
    depth = 5 if args.quick else 8
    cells, S = (2000, 64) if args.quick else (100000, 256)
    M.set_precision('tc_f16')
    nets = {
        'mega-nerf 8x256': O.make_net('mega', O.NerfSpec(), seed=3, n_sub=8, centroids=O.grid_centroids(2, 4), boundary_margin=1.15,
                                      cluster_2d=True),
        'nerf 2048 Cascade fine': O.make_net('cascade', O.NerfSpec(layer_dim=2048, appearance_dim=0), seed=3),
    }
    center, radius = [0.0, 0.0, 0.0], [0.6, 0.6, 0.6]
    rows_out = []
    for shape, net in nets.items():
        p = build_net(net, DEV)
        spec = net.spec
        hp = Namespace(init_grid_depth=depth, model_chunk_size=CHUNK, use_cascade=net.kind == 'cascade', samples_per_cell=S,
                       pos_dir_dim=spec.pos_dir_dim, appearance_dim=spec.appearance_dim, embedding_index=0, masking_mode='sigma')
        # thresholds at the 95th percentile of this net's densities: about 5% of the voxels are occupied
        off0, sc0 = MO.OT.box(center, radius)
        with torch.inference_mode():
            s0 = T.density_grid(p, off0, sc0, 64)
        q = float(torch.quantile(s0.cpu(), 0.95))
        hp.scale_alpha_thresh = MO.OT.alpha_for(q, 2 ** depth)
        hp.alpha_thresh = MO.OT.alpha_for(q, 2 ** (depth + 1))
        fl = trunk_flops_per_row(spec)

        # step 0
        rows = (2 ** depth) ** 3
        mult = multiplicity(net, off0, sc0)
        rec = Recorder(p)
        with torch.inference_mode():
            (rc, rr), ms_r, mem_r = timed(lambda: ref._auto_scale(hp, rec, list(center), list(radius), DEV))
            T.auto_scale(hp, p, center, radius, DEV)      # warm-up
            (oc, orad), ms_o, mem_o = timed(lambda: T.auto_scale(hp, p, center, radius, DEV))
        same = (rc, rr) == (oc, orad)
        rows_out.append(line('step0', shape, 'reference', ms_r, rows, fl, mult, mem_r))
        rows_out.append(line('step0', shape, 'octree', ms_o, rows, fl, mult, mem_o, box_equal=same, speedup=ms_r / ms_o))
        if net.kind != 'mega':
            continue

        # step 1 grid
        off1, sc1 = MO.OT.box(oc, orad)
        rows = (2 ** (depth + 1)) ** 3
        mult = multiplicity(net, off1, sc1)
        rec = Recorder(p)
        tree = MO.N3Tree(off1, sc1)
        err = None

        def ref_step1():
            try:
                ref._step1(hp, rec, tree, None, DEV)
            except RuntimeError as e:        # see DESIGN.md §7: the reference indexes its CPU lattice with a CUDA mask
                return str(e).splitlines()[0]
            return None
        with torch.inference_mode():
            err, ms_r, mem_r = timed(ref_step1)
            ref_sig = torch.cat(rec.kept)
            rec.kept = []
            T.grid_sigmas(hp, p, off1, sc1, DEV)
            (sig, pts), ms_o, mem_o = timed(lambda: (lambda s: (s, T.occupied_points(hp, s, off1, sc1)))(T.grid_sigmas(hp, p, off1, sc1, DEV)))
        same = torch.equal(sig, ref_sig)
        pts_same = torch.equal(pts, tree.refined[0]) if tree.refined else None
        rows_out.append(line('step1', shape, 'reference', ms_r, rows, fl, mult, mem_r, stopped_at=err))
        rows_out.append(line('step1', shape, 'octree', ms_o, rows, fl, mult, mem_o, sigmas_bit_equal=same, points_equal=pts_same,
                             occupied=int(pts.shape[0]), speedup=ms_r / ms_o))
        del ref_sig, sig, pts, tree

        # step 2
        g = torch.Generator(device=DEV).manual_seed(5)
        pts = torch.rand(cells, S, 3, generator=g, device=DEV) - 0.5
        rows = cells * S
        mult = multiplicity(net, torch.full((3,), 0.5), torch.ones(3))
        cells_ref = MO.N3Tree(off1, sc1, pts, spec.rgb_dim + 1)
        cells_new = MO.N3Tree(off1, sc1, pts, spec.rgb_dim + 1)

        def new_step2():
            cells_new[0:cells] = T.cell_colors(hp, p, pts).cpu()
        with torch.inference_mode():
            _, ms_r, mem_r = timed(lambda: ref._step2(hp, p, cells_ref, DEV))
            new_step2()
            _, ms_o, mem_o = timed(new_step2)
        d = float((cells_new.values - cells_ref.values).abs().max())
        rel = d / float(cells_ref.values.abs().max())
        rows_out.append(line('step2', shape, 'reference', ms_r, rows, fl, mult, mem_r))
        rows_out.append(line('step2', shape, 'octree', ms_o, rows, fl, mult, mem_o, rgba_max_abs_diff=d, rgba_rel_diff=rel,
                             speedup=ms_r / ms_o))
        del pts, cells_ref, cells_new
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=smi('name,power.limit,clocks.max.sm'), lines=rows_out), f, indent=1)


if __name__ == '__main__':
    main()
