"""CPU-only: the float64 stage restatement of tensor-core training (tests/tc_train_ref.py).

An fp32 emulation of the kernels (fp16 operands and images, fp32 accumulation in torch's summation order, which differs from
the float64 reference's) must pass every stage check at the shapes tests/test_gpu_zzc_train_tc_stages.py uses; each injected
bug must fail at least one stage; and without rounding the restatement is float64 autograd of the oracle's forward.  The same for
the forward stages and the output assembly alone (check_forward, check_output) at every shape tests/test_gpu_zzd_infer_tc.py
records, including the networks only tc_f16 inference runs."""
import pytest
import torch

import cases as C
import tc_train_ref as T
from oracle import mn_oracle as O


def emulate(spec, w, x, cot, noise, fused, bug=None):
    """What the kernels write for one sub-module's rows, in fp32 with fp16 rounding at the kernels' rounding points."""
    L, layers, in_xyz, R = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    half = L // 2
    f = lambda t: t.float()                                                           # noqa: E731
    h = lambda t: T.h16(t.float())                                                    # noqa: E731
    wf = {k: v.float() for k, v in w.items()}
    n = x.shape[0]
    pe = h(T.pe_band_fp32(x[:, :spec.xyz_dim], spec.pos_xyz_dim))
    aux = []
    if spec.pos_dir_dim > 0:
        aux.append(T.pe_band_fp32(x[:, -4:-1], spec.pos_dir_dim))
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    if ids is not None:
        aux.append(wf['embedding_a.weight'][ids])
    aux = h(torch.cat(aux, -1))
    img, pre_relu = [], []
    cur = pe
    for i in range(layers):
        if i in spec.skip_layers and i > 0:
            inp = torch.cat([cur, pe], -1) if bug == 'skip_swap' else torch.cat([pe, cur], -1)
        else:
            inp = cur
        a = inp @ h(wf[f'xyz_encodings.{i}.0.weight']).t() + wf[f'xyz_encodings.{i}.0.bias']
        pre_relu.append(torch.relu(a))
        cur = h(torch.relu(a))
        img.append(cur)
    H32 = pre_relu[-1] if fused else img[-1]
    sig = (H32 @ wf['sigma.weight'].t())[:, 0] + wf['sigma.bias'] + f(noise).view(-1)
    F_ = h(img[-1] @ h(wf['xyz_encoding_final.weight']).t() + wf['xyz_encoding_final.bias'])
    img.append(F_)
    G16 = h(torch.relu(torch.cat([F_, aux], -1) @ h(wf['dir_a_encoding.0.weight']).t() + wf['dir_a_encoding.0.bias']))
    img.append(G16)
    Wr = h(wf['rgb.weight']) if fused else wf['rgb.weight']
    lin = G16 @ Wr.t() + wf['rgb.bias']
    rgb = torch.sigmoid(lin) if R == 3 else lin[:, :3]
    S = T.grad_scale(cot)
    go = f(cot)
    if R == 3:
        d = (go[:, :3] * (1 - rgb)) * rgb
    else:
        d = go[:, :R]
    if spec.shifted_softplus:
        y = sig - 1
        dsp = torch.where(y > 20, torch.ones_like(y), 1 / (1 + torch.exp(-y)))
    else:
        dsp = (sig > 0).float()
    ds = go[:, R] * dsp
    gf32 = torch.cat([ds.view(-1, 1), d], 1)
    dzg32 = (d @ wf['rgb.weight']) * (G16 > 0)
    dz = {layers + 1: h(dzg32 * S)}
    dz[layers] = h(dz[layers + 1] @ h(wf['dir_a_encoding.0.weight'][:, :L]))
    dh = dz[layers] @ h(wf['xyz_encoding_final.weight']) + (ds * S).view(-1, 1) * wf['sigma.weight']
    dz[layers - 1] = h(dh * (img[layers - 1] > 0))
    for i in range(layers - 1, 0, -1):
        Wi = wf[f'xyz_encodings.{i}.0.weight']
        Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi
        mk = img[i] if (bug == 'mask_neighbour' and i == 3) else img[i - 1]
        dz[i - 1] = h((dz[i] @ h(Wh)) * (mk > 0))
    grads = {k: torch.zeros_like(v) for k, v in wf.items()}

    def wop(name, Z, X, s=S):
        keep = torch.ones(n, 1)
        if bug == 'dropped_tile' and name == 'xyz_encodings.2.0':
            keep[128:256] = 0
        grads[name + '.weight'] += ((Z * keep).t() @ X) / s
        grads[name + '.bias'] += (Z * keep).sum(0) / s

    FX = torch.cat([F_, aux], -1)
    wop('dir_a_encoding.0', dz[layers + 1], FX)
    wop('xyz_encoding_final', dz[layers], img[layers - 1])
    for i in range(layers):
        X = pe if i == 0 else img[i - 1]
        if i in spec.skip_layers and i > 0:
            X = torch.cat([pe, X], -1)
        wop(f'xyz_encodings.{i}.0', dz[i], X, S / 2 if (bug == 'scale_x2' and i == 1) else S)
        if bug == 'bias_segment' and i in spec.skip_layers and i > 0:     # the hidden segment's item owns the bias too
            grads[f'xyz_encodings.{i}.0.bias'] += dz[i].sum(0) / S
    grads['sigma.weight'] += ds.view(1, -1) @ img[layers - 1]
    grads['sigma.bias'] += ds.sum().view(1)
    grads['rgb.weight'] += d.t() @ G16
    grads['rgb.bias'] += d.sum(0)
    emb_sum = None
    if ids is not None:
        sid = ids + 1 if bug == 'emb_id' else ids
        emb_sum = torch.zeros(spec.appearance_count + 1, half).index_add_(0, sid, dzg32)[:spec.appearance_count]
        grads['embedding_a.weight'] += emb_sum @ wf['dir_a_encoding.0.weight'][:, L + spec.in_dir:]
    kpe = (in_xyz + 15) // 16 * 16
    xpe = torch.zeros(n, kpe)
    xpe[:, :in_xyz] = pe
    d64 = lambda t: t.double()                                                        # noqa: E731
    return dict(valid=torch.ones(n, dtype=torch.bool), x=d64(x), noise=d64(noise).view(-1), go=d64(cot),
                bw=torch.ones(n, dtype=torch.float64), xpe=d64(xpe), xaux=d64(aux), img=[d64(t) for t in img], sig=d64(sig),
                rgb=d64(rgb), id=d64(x[:, -1]) if ids is not None else torch.zeros(n, dtype=torch.float64), S=S,
                gf32=d64(gf32), dz={j: d64(t) for j, t in dz.items()},
                emb_sum=d64(emb_sum) if emb_sum is not None else None, grads={k: d64(v) for k, v in grads.items()})


SPECS = {
    'fused256_app': (O.NerfSpec(), True),
    'fused256_d12_sh2': (O.NerfSpec(layers=12, pos_dir_dim=0, rgb_dim=27), True),
    'fused512': (O.NerfSpec(layer_dim=512, appearance_dim=0), True),
    'layer768': (O.NerfSpec(layer_dim=768, appearance_dim=0), False),
    'layer2048_sh4': (O.NerfSpec(layer_dim=2048, pos_dir_dim=0, rgb_dim=75), False),
    'layer384': (O.NerfSpec(layer_dim=384, appearance_dim=0), False),
    'bg256': (O.NerfSpec(xyz_dim=4, shifted_softplus=False, skip_layers=(2, 5)), True),
}


def case(spec, n=384, seed=21):
    net = O.make_net('nerf', spec, seed=seed)
    if not spec.shifted_softplus:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
    x = C.nerf_rows(spec, n, 31)
    g = torch.Generator().manual_seed(5)
    cot = (torch.rand(n, spec.rgb_dim + 1, generator=g) - 0.3) * 1e-3
    noise = torch.randn(n, 1, generator=g)
    return net.weights[0], x, cot, noise


def stages(spec, w, cap, fused):
    rep = T.Report()
    with torch.no_grad():
        T.check_stages(spec, {k: v.double() for k, v in w.items()}, cap, fused, rep)
    return rep


@pytest.mark.parametrize('vname', list(SPECS))
def test_fp32_emulation_within_bounds(vname):
    spec, fused = SPECS[vname]
    w, x, cot, noise = case(spec, n=256 if spec.layer_dim >= 2048 else 384)
    with torch.no_grad():
        cap = emulate(spec, w, x, cot, noise, fused)
    rep = stages(spec, w, cap, fused)
    print(f'\n{vname}\n{rep.text()}')
    assert not rep.failures(), rep.failures()


BUGS = ['dropped_tile', 'bias_segment', 'scale_x2', 'skip_swap', 'mask_neighbour', 'emb_id']


@pytest.mark.parametrize('bug', BUGS)
def test_each_mutation_leaves_the_bounds(bug):
    spec, fused = SPECS['fused256_app']
    w, x, cot, noise = case(spec)
    with torch.no_grad():
        cap = emulate(spec, w, x, cot, noise, fused, bug)
    fails = stages(spec, w, cap, fused).failures()
    print(bug, [(r['stage'], r['fail']) for r in fails])
    assert fails, bug


def test_restatement_without_rounding_is_autograd():
    spec = O.NerfSpec()
    net = O.make_net('nerf', spec, seed=21)
    x = C.nerf_rows(spec, 200, 31)
    g = torch.Generator().manual_seed(5)
    cot = (torch.rand(200, 4, generator=g) - 0.3) * 1e-3
    noise = torch.rand(200, 1, generator=g)
    w = {k: v.double().requires_grad_(True) for k, v in net.weights[0].items()}
    out = O.nerf_forward(spec, w, x.double(), sigma_noise=noise.double())
    (out * cot.double()).sum().backward()
    with torch.no_grad():
        got = T.wide_tc_chain(spec, {k: v.detach() for k, v in w.items()}, x.double(), cot.double(), noise.double(), lambda t: t)
    for k, v in w.items():
        assert torch.allclose(got[k], v.grad, rtol=1e-9, atol=1e-15 * float(v.grad.abs().max())), k


def test_pe_band_error_within_pe_beta():
    """The fast encoder's double-angle recurrence stays within PE_BETA of the directly evaluated bands (the comment on pe_band
    in mn_mlp_tc.cu gives its size) over xyz in [-1, 1] and unit directions."""
    x = torch.linspace(-1, 1, 200001).view(-1, 1)
    for nf in (12, 4):
        got = T.pe_band_fp32(x, nf).double()
        want = O.embed(x.double(), nf)
        err = float((got - want).abs().max())
        print(f'pe_band, {nf} bands: max |error| {err:.2e}')
        assert err <= T.PE_BETA / 4, err


def test_half_ulp16():
    for v, want in ((1.0, 2.0 ** -11), (1.5, 2.0 ** -11), (2.0, 2.0 ** -10), (2.0 ** -14, 2.0 ** -25), (0.0, 2.0 ** -25),
                    (1e-6, 2.0 ** -25)):
        assert float(T.half_ulp16(torch.tensor([v]))) == want, v


# ------------------------------------------------------------------------------------------------------------------------
# the recording forward of every tensor-core network (tests/test_gpu_zzd_infer_tc.py) and its output assembly
# ------------------------------------------------------------------------------------------------------------------------
def emulate_forward(spec, w, x, noise, fused, bug=None):
    """The forward half of a capture for one sub-module's rows, and y [n, rgb_dim + 1]: the row's output before any blend
    weight, all in fp32 with fp16 rounding where the kernels round."""
    L, layers, in_xyz, R = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    h = lambda t: T.h16(t.float())                                                    # noqa: E731
    wf = {k: v.float() for k, v in w.items()}
    n = x.shape[0]
    pe = h(T.pe_band_fp32(x[:, :spec.xyz_dim], spec.pos_xyz_dim))
    aux = []
    if spec.pos_dir_dim > 0:
        aux.append(T.pe_band_fp32(x[:, -4:-1], spec.pos_dir_dim))
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    if T.app_in_dira(spec):
        aux.append(wf['embedding_a.weight'][ids])
    aux = h(torch.cat(aux, -1)) if aux else torch.zeros(n, 0)
    img, cur, last32 = [], pe, None
    for i in range(layers):
        inp = torch.cat([pe, cur], -1) if (i in spec.skip_layers and i > 0) else cur
        last32 = torch.relu(inp @ h(wf[f'xyz_encodings.{i}.0.weight']).t() + wf[f'xyz_encodings.{i}.0.bias'])
        cur = h(last32)
        img.append(cur)
    H32 = last32 if fused else img[-1]
    sig = (H32 @ wf['sigma.weight'].t())[:, 0] + wf['sigma.bias'] + noise.float().view(-1)
    if spec.has_dir_a:
        F_ = h(img[-1] @ h(wf['xyz_encoding_final.weight']).t() + wf['xyz_encoding_final.bias'])
        G16 = h(torch.relu(torch.cat([F_, aux], -1) @ h(wf['dir_a_encoding.0.weight']).t() + wf['dir_a_encoding.0.bias']))
        img += [F_, G16]
        src = G16
    else:             # the rgb head reads the last trunk image; the bug reads the (empty) G image of the record instead
        src = torch.zeros_like(img[-1]) if bug == 'head_reads_g' else img[-1]
    Wr = h(wf['rgb.weight']) if fused else wf['rgb.weight']
    lin = src @ Wr.t() + wf['rgb.bias']
    if spec.affine_appearance:
        Tm = (wf['embedding_a.weight'][ids] @ wf['affine.weight'].t() + wf['affine.bias']).view(-1, 3, 4)
        M3 = Tm[:, :, :3].transpose(1, 2) if bug == 'affine_transposed' else Tm[:, :, :3]
        lin = (M3 @ lin.unsqueeze(-1)).squeeze(-1) + Tm[:, :, 3]
    rgb = torch.sigmoid(lin) if R == 3 else lin
    if spec.shifted_softplus:
        sg = torch.nn.functional.softplus(sig if bug == 'softplus_unshifted' else sig - 1)
    else:
        sg = torch.relu(sig)
    kpe = (in_xyz + 15) // 16 * 16
    kaux = (aux.shape[1] + 15) // 16 * 16
    xpe, xaux = torch.zeros(n, kpe), torch.zeros(n, kaux)
    xpe[:, :in_xyz] = pe
    xaux[:, :aux.shape[1]] = aux
    tape_rgb = torch.zeros(n, 3) if spec.affine_appearance else rgb[:, :3]
    d64 = lambda t: t.double()                                                        # noqa: E731
    return dict(valid=torch.ones(n, dtype=torch.bool), x=d64(x), noise=d64(noise).view(-1), xpe=d64(xpe), xaux=d64(xaux),
                img=[d64(t) for t in img], sig=d64(sig), rgb=d64(tape_rgb),
                id=d64(x[:, -1]) if ids is not None else torch.zeros(n, dtype=torch.float64), y=torch.cat([rgb, sg.view(-1, 1)], 1))


_G = dict(layer_dim=64, appearance_count=10)
INFER_SPECS = {          # name: (spec, fused engine)
    'fused64': (O.NerfSpec(**_G), True),
    'fg128_l4': (O.NerfSpec(layer_dim=128, layers=4, skip_layers=(2,)), True),
    'fused192': (O.NerfSpec(layer_dim=192), True),
    'fused256_app': (O.NerfSpec(), True),
    'fused256_d12_sh2': (O.NerfSpec(layers=12, pos_dir_dim=0, rgb_dim=27), True),
    'affine': (O.NerfSpec(affine_appearance=True), True),
    'affine64': (O.NerfSpec(affine_appearance=True, **_G), True),
    'nodir_noapp': (O.NerfSpec(pos_dir_dim=0, appearance_dim=0), True),
    'nodir_noapp128': (O.NerfSpec(pos_dir_dim=0, appearance_dim=0, layer_dim=128), True),
    'noapp_q1': (O.NerfSpec(appearance_dim=0), True),
    'relu_sigma': (O.NerfSpec(shifted_softplus=False), True),
    'bg256': (O.NerfSpec(xyz_dim=4), True),
    'sh2': (O.NerfSpec(pos_dir_dim=0, rgb_dim=27), True),
    'fused512': (O.NerfSpec(layer_dim=512), True),
    'layer96': (O.NerfSpec(layer_dim=96), False),
    'layer160_nodir': (O.NerfSpec(layer_dim=160, pos_dir_dim=0, appearance_dim=0), False),
    'layer384': (O.NerfSpec(layer_dim=384, appearance_dim=0), False),
    'layer768': (O.NerfSpec(layer_dim=768, appearance_dim=0), False),
    'layer2048_sh4': (O.NerfSpec(layer_dim=2048, pos_dir_dim=0, rgb_dim=75), False),
}


def forward_case(spec, n=300, seed=21):
    net = O.make_net('nerf', spec, seed=seed)
    if not spec.shifted_softplus:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
    x = C.nerf_rows(spec, n, 31)
    noise = torch.randn(n, 1, generator=torch.Generator().manual_seed(5))
    return net.weights[0], x, noise


def forward_report(spec, w, cap, fused):
    rep = T.Report()
    wd = {k: v.double() for k, v in w.items()}
    with torch.no_grad():
        T.check_forward(spec, wd, cap, fused, rep)
        T.check_output(spec, cap['y'], [(torch.arange(cap['y'].shape[0]), None, T.slot_outputs(spec, wd, cap, fused))], rep)
    return rep


@pytest.mark.parametrize('vname', list(INFER_SPECS))
def test_forward_emulation_within_bounds(vname):
    spec, fused = INFER_SPECS[vname]
    w, x, noise = forward_case(spec, n=128 if spec.layer_dim >= 2048 else 300)
    with torch.no_grad():
        cap = emulate_forward(spec, w, x, noise, fused)
    rep = forward_report(spec, w, cap, fused)
    print(f'\n{vname}\n{rep.text()}')
    assert not rep.failures(), rep.failures()
    assert any(r['stage'] == 'out rgb' and r['n'] > 0 for r in rep.rows)


def routed_report(net, x, noise, bug=None):
    """A MegaNeRF call emulated per sub-module (ascending, or descending under the bug) with fp32 blending, then checked."""
    assign, wts = O.route(net, x)
    K, R = len(net.weights), net.spec.rgb_dim
    out = torch.zeros(x.shape[0], R + 1)
    per = {}
    with torch.no_grad():
        for s in range(K):
            rows = ((assign == s) if wts is None else (wts[:, s] > 0)).nonzero().view(-1)
            if len(rows):
                bw = wts[rows, s].float() if wts is not None else None
                per[s] = (rows, bw, emulate_forward(net.spec, net.weights[s], x[rows], noise[rows], True))
        for s in (sorted(per, reverse=True) if bug == 'combine_descending' else sorted(per)):
            rows, bw, cap = per[s]
            y = cap['y']
            if bw is not None:
                y = y * bw.view(-1, 1)
                if bug == 'slot_w_twice':
                    y = y * bw.view(-1, 1)
                out[rows] = out[rows] + y
            else:
                out[rows] = y
        rep = T.Report()
        pieces = []
        for s in sorted(per):
            rows, bw, cap = per[s]
            wd = {k: v.double() for k, v in net.weights[s].items()}
            T.check_forward(net.spec, wd, cap, True, rep, tag=f'[{s}] ')
            pieces.append((rows, bw, T.slot_outputs(net.spec, wd, cap, True)))
        T.check_output(net.spec, out, pieces, rep)
    return rep


@pytest.mark.parametrize('mname', ['hard2d', 'blend2d'])
def test_routed_emulation_within_bounds(mname):
    net = C.mega_net(mname)
    x = C.mega_rows(net, 1500, 13)
    noise = torch.rand(x.shape[0], 1, generator=torch.Generator().manual_seed(6))
    rep = routed_report(net, x, noise)
    print(f'\n{mname}\n{rep.text()}')
    assert not rep.failures(), rep.failures()


FWD_BUGS = {      # bug: the network it is injected into
    'affine_transposed': 'affine64',
    'slot_w_twice': 'blend2d',
    'combine_descending': 'blend2d',
    'softplus_unshifted': 'fused64',
    'head_reads_g': 'nodir_noapp128',
}


@pytest.mark.parametrize('bug', list(FWD_BUGS))
def test_each_forward_mutation_leaves_the_bounds(bug):
    where = FWD_BUGS[bug]
    if where in INFER_SPECS:
        spec, fused = INFER_SPECS[where]
        w, x, noise = forward_case(spec)
        with torch.no_grad():
            cap = emulate_forward(spec, w, x, noise, fused, bug)
        rep = forward_report(spec, w, cap, fused)
    else:
        net = C.mega_net(where)
        x = C.mega_rows(net, 1500, 13)
        rep = routed_report(net, x, torch.rand(x.shape[0], 1, generator=torch.Generator().manual_seed(6)), bug)
    fails = rep.failures()
    print(bug, [(r['stage'], r['fail']) for r in fails])
    assert fails, bug
