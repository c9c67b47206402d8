"""CPU: the float64 restatement of fp32 training (tests/fp32_train_ref.py) against an fp32 emulation of the kernels.

The emulation follows mlp_simt_kernel / mlp_bwd_data_kernel / mlp_bwd_weight_kernel step by step in float32 torch ops (tiles,
weight-gradient chunks, bucketed routing slots, blend weights, the ascending combine) and writes the same per-slot tapes, in a
channel layout of its own that it reports as the hook does.  Unchanged, it must pass every check at every shape of
tests/test_gpu_zze_train_fp32_stages.py; with one injected bug, the check named for that bug must fail."""
import pytest
import torch

import fp32_train_ref as R
import test_gpu_zze_train_fp32_stages as G
from oracle import mn_oracle as O

f = torch.float32


def tape_layout(spec):
    """Channel bases of the two tapes (the emulation's own; the GPU test reads the library's from the hook)."""
    L, layers = spec.layer_dim, spec.layers
    n_aux = spec.in_dir + (spec.appearance_dim if R.app_in_dira(spec) else 0)
    tl, c = {}, 0
    for k, n in (('a_pe', spec.in_xyz), ('a_aux', n_aux), ('a_h', layers * L), ('a_f', L), ('a_g', L // 2), ('a_rgb', spec.rgb_dim),
                 ('a_lin', 3), ('a_sig', 1), ('a_id', 1)):
        tl[k], c = c, c + n
    tl['a_total'] = c
    c = 0
    for k, n in (('g_z', layers * L), ('g_final', L), ('g_dira', L // 2), ('g_rgb', spec.rgb_dim), ('g_sig', 1)):
        tl[k], c = c, c + n
    tl['g_total'] = c
    tl['n_aux'] = n_aux
    return tl


def routing(net, x, TM):
    """Bucketed slots of a call as the router lays them out (rows ascending inside a bucket, where the GPU's order follows its
    atomics): slot_row, slot_w or None, bucket starts, sub-modules."""
    K = len(net.weights)
    if net.kind != 'mega':
        B = x.shape[0]
        S = -(-B // TM) * TM
        sr = torch.arange(S)
        sr[sr >= B] = -1
        return sr, None, [0, S], [0]
    assign, wts = O.route(net, x)
    mask = (torch.nn.functional.one_hot(assign, K) > 0) if wts is None else wts > 0
    counts = mask.sum(0)
    starts = [0]
    for k in range(K):
        starts.append(starts[-1] + int(-(-int(counts[k]) // R.MN_BUCKET) * R.MN_BUCKET))
    sr = torch.full((starts[-1],), -1, dtype=torch.long)
    sw = torch.zeros(starts[-1], dtype=torch.float64) if wts is not None else None
    for k in range(K):
        rows = torch.nonzero(mask[:, k]).view(-1)
        sr[starts[k]:starts[k] + len(rows)] = rows
        if sw is not None:
            sw[starts[k]:starts[k] + len(rows)] = wts[rows, k].double()
    return sr, sw, starts, list(range(K))


def forward_rows(spec, w, xs, noise, bugs):
    """The forward of rows xs through one sub-module in fp32: the tape blocks and the head values."""
    L, layers = spec.layer_dim, spec.layers
    pe = O.embed(xs[:, :spec.xyz_dim], spec.pos_xyz_dim)
    aux = []
    if spec.pos_dir_dim > 0:
        aux.append(O.embed(xs[:, -4:-1], spec.pos_dir_dim))
    ids = R.image_ids(spec, xs) if spec.appearance_dim > 0 else None
    if R.app_in_dira(spec):
        aux.append(w['embedding_a.weight'][ids])
    aux = torch.cat(aux, 1) if aux else pe[:, :0]
    h, cur = [], pe
    for i in range(layers):
        if i in spec.skip_layers and i > 0:
            cur = torch.cat([cur, pe], 1) if 'skip swapped' in bugs else torch.cat([pe, cur], 1)
        cur = torch.relu(cur @ w[f'xyz_encodings.{i}.0.weight'].t() + w[f'xyz_encodings.{i}.0.bias'])
        h.append(cur)
    t = dict(a_pe=pe, a_aux=aux, a_h=torch.cat(h, 1))
    sig = h[-1] @ w['sigma.weight'].t() + w['sigma.bias']
    if noise is not None:
        sig = sig + noise.view(-1, 1)
    t['a_sig'] = sig
    src = h[-1]
    if spec.has_dir_a:
        t['a_f'] = h[-1] @ w['xyz_encoding_final.weight'].t() + w['xyz_encoding_final.bias']
        t['a_g'] = src = torch.relu(torch.cat([t['a_f'], aux], 1) @ w['dir_a_encoding.0.weight'].t() + w['dir_a_encoding.0.bias'])
    lin = src @ w['rgb.weight'].t() + w['rgb.bias']
    rgb = lin
    if spec.affine_appearance and spec.appearance_dim > 0:
        t['a_lin'] = lin
        A = (w['embedding_a.weight'][ids] @ w['affine.weight'].t() + w['affine.bias']).view(-1, 3, 4)
        rgb = (A[:, :, :3] * lin.unsqueeze(1)).sum(-1) + A[:, :, 3]
    if spec.rgb_dim == 3:
        rgb = torch.sigmoid(rgb)
    t['a_rgb'] = rgb
    if ids is not None:
        t['a_id'] = ids.to(f).view(-1, 1)
    return t


def emulate(net, x, noise, go, TM=None, bugs=()):
    """-> a capture of fp32_train_ref, computed the kernels' way in fp32."""
    spec = net.spec
    L, layers, in_xyz, Rd = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    TM = TM or (64 if L <= 256 else 32)
    chunk = 64
    tl = tape_layout(spec)
    slot_row, slot_w, starts, subs = routing(net, x, TM)
    xc = x[:, 3:] if net.xyz_real else x
    S = len(slot_row)
    act = torch.zeros(S, tl['a_total'])
    grad = torch.zeros(S, tl['g_total'])
    K = len(net.weights)
    grads = [{k: torch.zeros_like(v) for k, v in w.items()} for w in net.weights]
    out = torch.zeros(x.shape[0], Rd + 1)
    blend = slot_w is not None
    for s, a, b in [(s, starts[i], starts[i + 1]) for i, s in enumerate(subs)]:
        idx = torch.arange(a, b)
        val = slot_row[a:b] >= 0
        if not bool(val.any()):
            continue
        sl = idx[val]
        rows = slot_row[sl]
        w = net.weights[s]
        xs = xc[rows]
        nz = noise.view(-1)[rows] if noise is not None else None
        t = forward_rows(spec, w, xs, nz, bugs)
        if 'neighbour weights' in bugs:              # the first tile of the bucket runs through sub-module s + 1
            first = sl < a + TM
            tn = forward_rows(spec, net.weights[(s + 1) % K], xs[first], nz[first] if nz is not None else None, bugs)
            for k in t:
                t[k][first] = tn[k]
        for k, v in t.items():
            act[sl, tl[k]:tl[k] + v.shape[1]] = v
        # ---- out
        sig = torch.nn.functional.softplus(t['a_sig'] - 1, 1, 20) if spec.shifted_softplus else torch.relu(t['a_sig'])
        o = torch.cat([t['a_rgb'], sig], 1)
        if blend:
            out[rows] = out[rows] + o * slot_w[sl].to(f).view(-1, 1)
        else:
            out[rows] = o
        # ---- data gradients
        GO = go[rows].to(f)
        if blend and 'no blend weight' not in bugs:
            GO = GO * slot_w[sl].to(f).view(-1, 1)
        pre = t['a_sig'][:, 0]
        if spec.shifted_softplus:
            y = pre if 'unshifted softplus' in bugs else pre - 1
            d = torch.where(y > 20, torch.ones_like(y), torch.sigmoid(y))
        else:
            d = (pre > 0).to(f)
        DS = (GO[:, Rd] * d).view(-1, 1)
        dv = (GO[:, :Rd] * (1 - t['a_rgb'])) * t['a_rgb'] if Rd == 3 else GO[:, :Rd]
        DR = dv
        g = {'g_sig': DS}
        ids = R.image_ids(spec, xs) if spec.appearance_dim > 0 else None
        if spec.affine_appearance and spec.appearance_dim > 0:
            e = w['embedding_a.weight'][ids]
            A = (e @ w['affine.weight'].t() + w['affine.bias']).view(-1, 3, 4)
            DR = (A[:, :, :3] * dv.unsqueeze(-1)).sum(1)
            lin = t['a_lin']
            if 'dA transposed' in bugs:
                dA = torch.cat([dv.unsqueeze(1) * lin.unsqueeze(-1), dv.unsqueeze(-1)], -1).view(-1, 12)
            else:
                dA = torch.cat([dv.unsqueeze(-1) * lin.unsqueeze(1), dv.unsqueeze(-1)], -1).view(-1, 12)
            gw = grads[s]
            gw['affine.bias'] += dA.sum(0)
            gw['affine.weight'] += dA.t() @ e
            gw['embedding_a.weight'].index_add_(0, ids, dA @ w['affine.weight'])
        g['g_rgb'] = DR
        H = t['a_h'][:, (layers - 1) * L:]
        addw = 'no addw' not in bugs
        if spec.has_dir_a:
            dzg = (DR @ w['rgb.weight']) * (t['a_g'] > 0)
            g['g_dira'] = dzg
            g['g_final'] = dzf = dzg @ w['dir_a_encoding.0.weight'][:, :L]
            if R.app_in_dira(spec):
                eid = (ids + 1) % spec.appearance_count if 'embedding id+1' in bugs else ids
                grads[s]['embedding_a.weight'].index_add_(0, eid, dzg @ w['dir_a_encoding.0.weight'][:, L + spec.in_dir:])
            dz = dzf @ w['xyz_encoding_final.weight']
        else:
            dz = DR @ w['rgb.weight']
        if addw:
            dz = dz + DS * w['sigma.weight']
        dz = dz * (H > 0)
        dzs = [None] * layers
        dzs[layers - 1] = dz
        for i in range(layers - 1, 0, -1):
            Wi = w[f'xyz_encodings.{i}.0.weight']
            Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi
            m = t['a_h'][:, i * L:(i + 1) * L] if 'mask from the wrong layer' in bugs else t['a_h'][:, (i - 1) * L:i * L]
            dzs[i - 1] = (dzs[i] @ Wh) * (m > 0)
        g['g_z'] = torch.cat(dzs, 1)
        for k, v in g.items():
            grad[sl, tl[k]:tl[k] + v.shape[1]] = v
    # ---- weight gradients: per sub-module, per chunk of `chunk` tiles, then the chunks added
    cap = dict(TM=TM, chunk=chunk, tl=tl, act=act.double(), grad=grad.double(), slot_row=slot_row, n_slots=S, slot_w=slot_w,
               starts=starts, subs=subs, x=xc, noise=noise.view(-1) if noise is not None else None, go=go, out=out, grads=None)
    for s, a, b in R.sub_ranges(cap):
        c = R.restrict(dict(cap, act=act, grad=grad), a, b)
        gw = grads[s]
        t0 = 1 if 'chunk start off by one' in bugs else 0
        tiles = (b - a) // TM
        for name, Z, X in R.linear_ops(spec, c):
            kblocks = -(-X.shape[1] // 64)
            for c0 in range(t0, tiles, chunk):
                c1 = min(tiles, c0 + chunk) - (1 if 'drop last tile' in bugs else 0)
                z, xx = Z[c0 * TM:c1 * TM], X[c0 * TM:c1 * TM]
                gw[name + '.weight'] += z.t() @ xx
                gw[name + '.bias'] += z.sum(0) * (kblocks if 'bias on every k block' in bugs else 1)
    cap['grads'] = [{k: v.double() for k, v in gw.items()} for gw in grads]
    return cap


def case_rows(vname, n):
    spec = G.SPECS[vname]
    x, cot, noise = G.rows_and_grads(spec, n, 5)
    return G.make(spec), x, cot, noise


def run_checks(net, x, noise, cot, bugs=()):
    cap = emulate(net, x, noise, cot, bugs=bugs)
    rep = R.Report()
    R.check_call(net.spec, net.weights, cap, rep)
    return rep


@pytest.mark.parametrize('vname', list(G.SPECS))
def test_emulation_passes(vname):
    net, x, cot, noise = case_rows(vname, 200)
    rep = run_checks(net, x, noise, cot)
    assert not rep.failures(), rep.text()


@pytest.mark.parametrize('vname,n', [('w192', 129), ('w192', G.chunks3(64)), ('w448', G.chunks3(32))])
def test_emulation_passes_many_chunks(vname, n):
    net, x, cot, noise = case_rows(vname, n)
    rep = run_checks(net, x, noise, cot)
    assert not rep.failures(), rep.text()


@pytest.mark.parametrize('mname', list(G.MEGA))
def test_emulation_passes_routed(mname):
    net, x, cot, noise = G.mega_case(mname)
    rep = run_checks(net, x, noise, cot)
    assert not rep.failures(), rep.text()


def test_probe_emulation_exact():
    """A one-hot grad_out through the emulation: the probe checks hold bit for bit (torch's fp32 products are the kernels')."""
    net, x, cot, noise = case_rows('w192', G.chunks3(64))
    for row in (64 * 64, R.MN_BUCKET - 1, x.shape[0] - 1):
        g = torch.zeros_like(cot)
        g[row] = cot[row]
        rep = R.Report()
        R.check_probe(net.spec, emulate(net, x, noise, g), row, rep)
        assert not rep.failures(), rep.text()


BUGS = {
    # bug: (case, a stage that must fail)
    'drop last tile': ('w192_chunks', 'grad xyz_encodings.3.0.weight'),
    'bias on every k block': ('w192', 'grad xyz_encodings.3.0.bias'),
    'chunk start off by one': ('w192_chunks', 'grad xyz_encodings.3.0.weight'),
    'neighbour weights': ('blend8', 'fwd h0'),
    'mask from the wrong layer': ('w192', 'bwd dZ_2'),
    'skip swapped': ('w192', 'fwd h4'),
    'no addw': ('w192', 'bwd dZ_7'),
    'unshifted softplus': ('w192', 'bwd dsigma'),
    'embedding id+1': ('w192', 'grad embedding_a.weight'),
    'no blend weight': ('blend8', 'bwd dsigma'),
    'dA transposed': ('affine192', 'grad affine.weight'),
}


@pytest.mark.parametrize('bug', list(BUGS))
def test_injected_bug_fails(bug):
    case, stage = BUGS[bug]
    if case in G.MEGA:
        net, x, cot, noise = G.mega_case(case)
    elif case == 'w192_chunks':
        net, x, cot, noise = case_rows('w192', G.chunks3(64))
    else:
        net, x, cot, noise = case_rows(case, 300)
    rep = run_checks(net, x, noise, cot, bugs=(bug,))
    failed = [r['stage'] for r in rep.failures()]
    assert any(f.split('] ')[-1] == stage for f in failed), (bug, failed)
