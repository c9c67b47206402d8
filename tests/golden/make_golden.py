"""Generate tests/golden/hotpath_v1.pt by running the UNMODIFIED reference (imported read-only
from $MEGA_NERF_REFERENCE) on the seeded cases of tests/cases.py.

Needs a checkout of the reference:
    MEGA_NERF_REFERENCE=<path> python tests/golden/make_golden.py
The reference has no tests or golden vectors of its own (SURVEY.md §4); these fixtures are what
pins the oracle (oracle/mn_oracle.py) and, through it, the CUDA path.
"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
REF = os.environ['MEGA_NERF_REFERENCE']     # a checkout of the reference repository
sys.path.insert(0, REF)

import cases as C  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

from mega_nerf import ray_utils as R_rays  # noqa: E402
from mega_nerf import rendering as R_render  # noqa: E402
from mega_nerf.spherical_harmonics import eval_sh as R_eval_sh  # noqa: E402
from mega_nerf.models.nerf import NeRF as R_NeRF, ShiftedSoftplus as R_SSP, Embedding as R_Embedding  # noqa: E402
from mega_nerf.models.mega_nerf import MegaNeRF as R_MegaNeRF  # noqa: E402
from mega_nerf.models.cascade import Cascade as R_Cascade  # noqa: E402


def ref_nerf(spec: O.NerfSpec, w) -> nn.Module:
    m = R_NeRF(spec.pos_xyz_dim, spec.pos_dir_dim, spec.layers, list(spec.skip_layers), spec.layer_dim,
               spec.appearance_dim, spec.affine_appearance, spec.appearance_count, spec.rgb_dim, spec.xyz_dim,
               R_SSP() if spec.shifted_softplus else nn.ReLU())
    m.load_state_dict(w)
    return m.eval()


def ref_net(net: O.Net) -> nn.Module:
    subs = [ref_nerf(net.spec, w) for w in net.weights]
    if net.kind == 'nerf':
        return subs[0]
    if net.kind == 'cascade':
        return R_Cascade(subs[0], subs[1]).eval()
    return R_MegaNeRF(subs, net.centroids, net.boundary_margin, net.xyz_real, net.cluster_2d).eval()


def hparams_of(opts: O.RenderOpts) -> Namespace:
    return Namespace(**vars(opts))


def main():
    torch.manual_seed(1234)
    G = {}
    worst = 0.0

    def cmp(name, a, b):
        nonlocal worst
        d = float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
        worst = max(worst, d)
        if d != 0.0:
            print(f'  oracle != reference on {name}: max abs diff {d:.3e}')

    with torch.inference_mode():
        # ---- seeded init reproduces the reference constructor's RNG consumption
        for vname, v in C.NERF_VARIANTS.items():
            spec = v['spec']
            torch.manual_seed(77)
            ref = R_NeRF(spec.pos_xyz_dim, spec.pos_dir_dim, spec.layers, list(spec.skip_layers), spec.layer_dim,
                         spec.appearance_dim, spec.affine_appearance, spec.appearance_count, spec.rgb_dim,
                         spec.xyz_dim, R_SSP() if spec.shifted_softplus else nn.ReLU())
            torch.manual_seed(77)
            mine = O.init_nerf_weights(spec)
            sd = ref.state_dict()
            assert set(sd) == set(mine), (vname, set(sd) ^ set(mine))
            for k in sd:
                assert torch.equal(sd[k], mine[k]), (vname, k)

        # ---- ray generation
        for cp in (True, False):
            d = R_rays.get_ray_directions(13, 7, 9.5, 9.1, 6.2, 3.4, cp, torch.device('cpu'))
            G[f'raydirs_cp{int(cp)}'] = d.clone()
            cmp('raydirs', d, O.ray_directions(13, 7, 9.5, 9.1, 6.2, 3.4, cp))
        g = torch.Generator().manual_seed(5)
        q, _ = torch.linalg.qr(torch.randn(4, 3, 3, generator=g))
        c2w = torch.cat([q, torch.tensor([[-0.4, 0.1, 0.2], [-0.1, 0.0, 0.3], [-0.6, -0.2, 0.1], [0.1, 0.2, 0.3]]).unsqueeze(-1)], -1)
        dirs = O.ray_directions(13, 7, 9.5, 9.1, 6.2, 3.4, True)
        for alt in (None, [-0.35, 0.05]):
            tag = 'alt' if alt is not None else 'noalt'
            r = R_rays.get_rays(dirs, c2w[0], 0.1, 3.0, alt)
            G[f'rays_{tag}'] = r.clone()
            cmp('rays', r, O.rays_from_pose(dirs, c2w[0], 0.1, 3.0, alt))
            rb = R_rays.get_rays_batch(dirs.view(1, -1, 3).expand(4, -1, -1).contiguous(), c2w, 0.1, 3.0, alt)
            G[f'rays_batch_{tag}'] = rb.clone()
            cmp('rays_batch', rb, O.rays_from_pose_batch(dirs.view(1, -1, 3).expand(4, -1, -1).contiguous(), c2w, 0.1, 3.0, alt))
        G['raygen_c2w'] = c2w

        # ---- positional encoding
        for dim, L in ((3, 12), (4, 12), (3, 4)):
            gg = torch.Generator().manual_seed(dim * 100 + L)
            x = torch.rand(257, dim, generator=gg) * 2 - 1
            e = R_Embedding(L)(x)
            G[f'embed_d{dim}_L{L}'] = e.clone()
            cmp('embed', e, O.embed(x, L))

        # ---- single MLP variants
        for vname, v in C.NERF_VARIANTS.items():
            spec = v['spec']
            net = O.make_net('nerf', spec, seed=21)
            x = C.nerf_rows(spec, 160, 31)
            ref = ref_nerf(spec, net.weights[0])
            y = ref(x)
            G[f'nerf_{vname}'] = dict(out=y.clone(), wsum=C.net_checksum(net), xsum=C.checksum(x))
            cmp(f'nerf_{vname}', y, O.nerf_forward(spec, net.weights[0], x))
            xs = C.nerf_rows(spec, 160, 31, sigma_only=True)
            ys = ref(xs, sigma_only=True)
            G[f'nerf_{vname}']['sigma_only'] = ys.clone()
            cmp(f'nerf_{vname}_sigma', ys, O.nerf_forward(spec, net.weights[0], xs, sigma_only=True))
            gg = torch.Generator().manual_seed(41)
            noise = torch.rand(160, 1, generator=gg)
            yn = ref(x, sigma_noise=noise)
            G[f'nerf_{vname}']['noise_out'] = yn.clone()
            cmp(f'nerf_{vname}_noise', yn, O.nerf_forward(spec, net.weights[0], x, sigma_noise=noise))

        # ---- router / blender
        for mname in C.MEGA_VARIANTS:
            net = C.mega_net(mname)
            x = C.mega_rows(net, 700, 51)
            ref = ref_net(net)
            y = ref(x)
            assign, wts = O.route(net, x)
            G[f'mega_{mname}'] = dict(out=y.clone(), wsum=C.net_checksum(net), xsum=C.checksum(x),
                                      assign=assign, weights=wts)
            cmp(f'mega_{mname}', y, O.mega_forward(net, x))

        # ---- SH
        gg = torch.Generator().manual_seed(61)
        dirs_sh = torch.randn(300, 3, generator=gg)
        dirs_sh = dirs_sh / dirs_sh.norm(dim=-1, keepdim=True)
        for deg in range(5):
            sh = torch.randn(300, 3, (deg + 1) ** 2, generator=gg)
            y = R_eval_sh(deg, sh, dirs_sh)
            G[f'sh_deg{deg}'] = y.clone()
            cmp(f'sh{deg}', y, O.eval_sh(deg, sh, dirs_sh))

        # ---- stratified jitter (injected rand), resampling, compositing
        gg = torch.Generator().manual_seed(71)
        n, s = 200, 64
        near = torch.rand(n, 1, generator=gg) * 0.1 + 0.01
        far = near + torch.rand(n, 1, generator=gg) + 0.2
        t = torch.linspace(0, 1, s)
        z0 = near * (1 - t) + far * t
        rnd = torch.rand(n, s, generator=gg)
        torch.manual_seed(9)
        zj_ref = R_render._expand_and_perturb_z_vals(z0, s, 1.0, n)
        torch.manual_seed(9)
        rr = torch.rand(n, s)
        G['stratify_globalrng'] = zj_ref.clone()
        cmp('stratify', zj_ref, O.stratify(z0, s, 1.0, n, rand=rr))
        zj = O.stratify(z0, s, 1.0, n, rand=rnd)
        G['stratify_injected'] = zj.clone()

        sig = torch.rand(n, s, generator=gg) * 30 * (torch.rand(n, s, generator=gg) > 0.5)
        rgb = torch.rand(n, s, 3, generator=gg)
        ld = torch.full((n, 1), 1e10)
        ld[::3, 0] = torch.rand((n + 2) // 3, generator=gg)
        for flip in (False, True):
            zz = torch.flip(zj, dims=[-1]) if flip else zj
            res = {}
            R_render._inference  # (composite tail is exercised through render cases; here the oracle's own)
            c = O.composite(rgb, sig, zz, ld, flip, None)
            # reference tail, restated call-by-call through its public pieces is not exposed; check via
            # a stub network that returns (rgb, sigma) verbatim:

            class Stub(nn.Module):
                def __init__(self):
                    super().__init__()
                    self.k = 0

                def forward(self, x, sigma_only=False, sigma_noise=None):
                    out = torch.cat([rgb.view(-1, 3), sig.view(-1, 1)], 1)
                    return out

            hp = Namespace(pos_dir_dim=4, sh_deg=None, model_chunk_size=1 << 30, use_cascade=False)
            stub = Stub().eval()
            xyz = torch.zeros(n, s, 3)
            R_render._inference(results=res, typ='coarse', nerf=stub, rays_d=torch.zeros(n, 1, 3), image_indices=None,
                                hparams=hp, xyz=xyz, z_vals=torch.flip(zz, dims=[-1]) if flip else zz, last_delta=ld,
                                composite_rgb=True, get_depth=True, get_depth_variance=True, get_weights=True,
                                get_bg_lambda=True, flip=flip, depth_real=None)
            tag = f'composite_flip{int(flip)}'
            G[tag] = {k: v.clone() for k, v in res.items()}
            cmp(tag + '_w', res['weights_coarse'], c['weights'])
            cmp(tag + '_rgb', res['rgb_coarse'], c['rgb'])
            cmp(tag + '_d', res['depth_coarse'], c['depth'])
            cmp(tag + '_v', res['depth_variance_coarse'], c['depth_variance'])
            cmp(tag + '_l', res['bg_lambda_coarse'], c['bg_lambda'])

        w_coarse = O.composite(rgb, sig, zj, ld, False)['weights']
        mid = 0.5 * (zj[:, :-1] + zj[:, 1:])
        zf = R_render._sample_pdf(mid, w_coarse[:, 1:-1], 128, det=True)
        zo, cdf = O.sample_pdf(mid, w_coarse[:, 1:-1], 128, True, return_cdf=True)
        _, inds = O.sample_cdf(mid, cdf, 128, True, return_inds=True)
        G['resample_det'] = dict(z=zf.clone(), cdf=cdf.clone(), inds=inds.clone())
        cmp('resample_det', zf, zo)
        u = torch.rand(n, 128, generator=gg)
        torch.manual_seed(13)
        zr = R_render._sample_pdf(mid, w_coarse[:, 1:-1], 128, det=False)
        torch.manual_seed(13)
        u_g = torch.rand(n, 128)
        cmp('resample_rand', zr, O.sample_pdf(mid, w_coarse[:, 1:-1], 128, False, u=u_g))
        zu, inds_u = O.sample_cdf(mid, cdf, 128, False, u=u, return_inds=True)
        G['resample_u'] = dict(z=zu.clone(), inds=inds_u.clone())
        G['resample_inputs_sum'] = C.checksum(zj, sig, rgb, ld, u)

        # ---- background geometry
        rays_bg = O.synthetic_rays(150, seed=3, far=1e5)
        center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
        ff = R_render._intersect_sphere(rays_bg[:, :3], rays_bg[:, 3:6], center, radius)
        G['bg_fg_far'] = ff.clone()
        cmp('intersect', ff, O.intersect_sphere(rays_bg[:, :3], rays_bg[:, 3:6], center, radius))
        bz = O.stratify(torch.linspace(0, 1, 32), 32, 1.0, 150, rand=torch.rand(150, 32, generator=gg))
        for real, c2d in ((False, False), (True, True), (True, False)):
            p, dr = R_render._depth2pts_outside(rays_bg[:, None, :3], rays_bg[:, None, 3:6], bz, center, radius, real, c2d)
            G[f'bg_pts_real{int(real)}_2d{int(c2d)}'] = dict(pts=p.clone(), depth_real=dr.clone())
            po, dro = O.points_outside(rays_bg[:, None, :3], rays_bg[:, None, 3:6], bz, center, radius, real, c2d)
            cmp('bgpts', p, po)
            cmp('bgdr', dr, dro)
        G['bg_z'] = bz.clone()

        # ---- render_rays end to end
        for rname in C.RENDER_CASES:
            net, bg_net, rays, idx, opts, center, radius = C.render_case(rname)
            rn, rb = ref_net(net), (ref_net(bg_net) if bg_net is not None else None)
            hp = hparams_of(opts)
            res, present = R_render.render_rays(rn, rb, rays, idx, hp, center, radius, True, True, True)
            ores, opresent = O.render_rays(net, bg_net, rays, idx, opts, center, radius, True, True, True)
            assert set(res) == set(ores), (rname, set(res) ^ set(ores))
            assert present == opresent
            for k in res:
                cmp(f'render_{rname}_{k}', res[k], ores[k])
            G[f'render_{rname}'] = dict(out={k: v.clone() for k, v in res.items()}, present=present,
                                        wsum=C.net_checksum(net) + (C.net_checksum(bg_net) if bg_net else 0.0),
                                        xsum=C.checksum(rays, idx))
            print(f'render_{rname}: keys={sorted(res)} present={present}')

    C.save_golden(G, C.GOLDEN_PATH)
    print(f'wrote {C.GOLDEN_PATH}.part*; worst oracle-vs-reference diff {worst:.3e}')


if __name__ == '__main__':
    main()
