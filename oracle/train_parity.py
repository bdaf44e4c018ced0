"""Oracle-side parity report for the training-form render and its backward (test infrastructure, see oracle/__init__.py).

The training counterpart of ``parity.render_parity``, with the same three-part rule:

  (a) geometry   : the kernel's sample coordinates (``so_render_train_probe``) equal the fp64 oracle's within rounding;
  (b) same cells : the differentiable fp64 oracle evaluated AT the forward's fp32 coordinates vs the kernel -- per-sample
                   outputs, per-ray outputs, the max-depth index and the gradients w.r.t. the volume and inv_s, on every ray;
  (c) independent: the plain fp64 oracle vs the kernel on every ray without a cell flip; every ray whose depth misses
                   ``tol`` must contain a flip (attributed, never waved through), and flip rays are counted and bounded.

The analytic sdf gradient jumps across cell faces, so a gradient is only comparable where both sides differentiate the same
function: the caller zeroes the cotangents of every ray flagged by ``flip_rays`` (a sample whose cell differs between the
kernel and the fp64 evaluation) on both sides before the backward runs.
"""
import torch

from . import render as orender
from .parity import _idx_report

# kernel output name -> oracle output name
PER_SAMPLE = (('weights', 'weights'), ('ts', 'ts'), ('deltas', 'deltas'), ('eik_grad', 'eik_grad'), ('sample_sdf', 'sdf'))
PER_RAY = (('depth', 'depth'), ('acc', 'accumulation'), ('fars', 'fars'), ('rgb', 'rgb'), ('sem', 'sem'))
# differentiable outputs that take a cotangent
DIFF = ('depth', 'acc', 'weights', 'eik_grad', 'sample_sdf', 'rgb', 'sem')
# (atol, rtol) of test_render_train_forward_backward (tests/test_gpu_train.py)
TOL = {'weights': (2e-6, 1e-4), 'ts': (1e-5, 1e-5), 'deltas': (4e-6, 1e-4), 'eik_grad': (2e-5, 1e-4), 'sample_sdf': (2e-5, 1e-4),
       'depth': (1e-5, 1e-4), 'acc': (2e-5, 1e-4), 'fars': (1e-5, 1e-4), 'rgb': (5e-5, 1e-4), 'sem': (5e-5, 1e-4)}


def sample_geometry(mapping, o, d, aabb, S, jitter=None, near_plane=0.0, anchor='mid'):
    """fp64 grid coordinates [n, S, 3] of every training sample, and the (lo, hi) expected-depth clip bounds of the whole
    batch (the kernels take one clip over every ray of a launch; a chunked oracle must use the same bounds)."""
    nears, fars = orender.aabb_near_far(o, d, aabb, near_plane, True)
    starts, ends = orender.uniform_bins(nears, fars, S, jitter)
    mids = (starts + ends) / 2
    tq = mids if anchor == 'mid' else starts
    grid = mapping.meter2grid(o[:, None, :] + d[:, None, :] * tq[..., None], False)
    return grid, (mids.min(), mids.max())


def flip_rays(grid, *others):
    """bool [n]: rays with a sample whose cell (floor of any grid coordinate) differs between ``grid`` and any of ``others``."""
    n = grid.shape[0]
    cell = grid.double().floor()
    out = torch.zeros(n, dtype=torch.bool, device=grid.device)
    for g in others:
        out |= (g.double().to(grid.device).floor() != cell).reshape(n, -1).any(-1)
    return out


def oracle_train(vol64, mapping, o, d, nrm, aabb, inv_s, S, cot, jitter=None, color_dims=0, bkgd_rand=None, grid_override=None,
                 depth_clip=None, chunk=512, extra=None, **kw):
    """Differentiable fp64 oracle over ray chunks: returns (outputs in kernel names, d/d vol [Cf,H,W,Z], d/d inv_s,
    sum over samples of |per-sample term of d/d inv_s|) where the gradients are those of sum_k <output_k, cot[k]>
    (missing cotangents = zero).  ``extra(sl, named)`` -> (loss term, {name: per-ray tensor}) adds terms computed from a
    chunk's outputs (rays ``sl``) to its loss and outputs (train_objective.py)."""
    vol = vol64.detach().clone().requires_grad_(True)
    invs = torch.tensor(float(inv_s), dtype=torch.float64, device=vol.device, requires_grad=True)
    n = o.shape[0]
    outs, mass = {}, 0.0
    for b in range(0, n, chunk):
        sl = slice(b, min(b + chunk, n))
        iv = invs.expand(sl.stop - sl.start, S).clone()    # one inv_s per sample: its gradient is that sample's term
        iv.retain_grad()
        r = orender.neus_render_chunk(vol, mapping, o[sl], d[sl], nrm[sl], aabb, iv, S=S, training=True,
                                      jitter=None if jitter is None else jitter[sl], color_dims=color_dims,
                                      bkgd='random' if bkgd_rand is not None else 'white',
                                      bkgd_rand=None if bkgd_rand is None else bkgd_rand[sl], differentiable=True,
                                      grid_override=None if grid_override is None else grid_override[sl],
                                      depth_clip=depth_clip, **kw)
        r['ts'] = (r['starts'] + r['ends']) / 2 / nrm[sl]
        r['deltas'] = (r['ends'] - r['starts']) / nrm[sl]
        named = {k: r[rk] for k, rk in PER_SAMPLE + PER_RAY if rk in r}
        loss = sum((named[k] * cot[k][sl].to(named[k])).sum() for k in DIFF if k in cot and k in named)
        if extra is not None:
            term, more = extra(sl, named)
            loss = loss + term
            named.update(more)
        loss.backward()
        mass += float(iv.grad.abs().sum()) if iv.grad is not None else 0.0      # None: no term depends on inv_s
        for k, t in named.items():
            outs.setdefault(k, []).append(t.detach())
    outs = {k: torch.cat(v) for k, v in outs.items()}
    outs['max_depth'], outs['max_idx'] = orender.max_depth_ref(outs['weights'], outs['ts'], outs['deltas'])
    return outs, vol.grad, invs.grad, mass


def _close(a, b, atol, rtol, rows=None):
    """(max |a - b| / (atol + rtol |b|), max |a - b|) over the selected rays; <= 1 passes."""
    a, b = a.double().reshape(b.shape).to(b.device), b.double()
    if rows is not None:
        a, b = a[rows], b[rows]
    if a.numel() == 0:
        return 0.0, 0.0
    e = (a - b).abs()
    return float((e / (atol + rtol * b.abs())).max()), float(e.max())


# The fp32 error of everything computed from alpha (weights, per-ray sums, gradients) is the error of the alpha argument
# inv_s * (sdf -+ half), half = min(tc, 0) * delta / 2, times a sensitivity of order one.  The tolerances of TOL were set
# where inv_s times the field's fp32 error is about A0 (tests/test_gpu_train.py: inv_s 12, |d sdf| + |d half| ~ 1e-6);
# elsewhere they are scaled by kappa = max(1, inv_s * err / A0), with err measured on the case itself.
A0 = 1.2e-5
SCALED = ('weights', 'depth', 'acc', 'rgb', 'sem', 'grad_sdf', 'grad_feat', 'grad_inv_s')


def alpha_arg_error(got, ref, d, nrm, rows=None):
    """max over samples of |d sdf| + |d half| (metres) between the kernel's fp32 field / geometry and ``ref``."""
    n, S = got['weights'].shape[0], got['weights'].reshape(got['weights'].shape[0], -1).shape[1]
    dev = ref['sdf'].device if 'sdf' in ref else ref['sample_sdf'].device
    sdf_k, sdf_r = got['sample_sdf'].double().to(dev).reshape(n, S), ref['sample_sdf'].reshape(n, S)
    eik_k, eik_r = got['eik_grad'].double().to(dev).reshape(n, S, 3), ref['eik_grad'].reshape(n, S, 3)
    dl_k, dl_r = got['deltas'].double().to(dev).reshape(n, S) * nrm, ref['deltas'].reshape(n, S) * nrm
    tc_r = (eik_r * d[:, None, :]).sum(-1)
    err = (sdf_k - sdf_r).abs() + 0.5 * ((dl_k - dl_r).abs() * tc_r.abs() + dl_r.abs() * (eik_k - eik_r).norm(dim=-1))
    if rows is not None:
        err = err[rows]
    return float(err.max()) if err.numel() else 0.0


def _compare(got, ref, grads, gref, n, S, kappa, deltas_atol, rows=None):
    rep = {}
    for k, _ in PER_SAMPLE + PER_RAY:
        if k in got and k in ref and got[k] is not None and got[k].numel():
            atol, rtol = TOL[k]
            if k == 'deltas':
                atol = max(atol, deltas_atol)
            if k in SCALED:
                atol, rtol = atol * kappa, rtol * kappa
            rep[k] = _close(got[k], ref[k], atol, rtol, rows)
    # max depth: the kernel returns ts at its index.  Rays whose max depth equals the oracle's within the ts tolerance agree
    # (this covers rays that miss the AABB, whose samples all have zero length); on the others ts increase strictly along
    # the ray, the kernel's index is recovered exactly and must pass the tie rule of the inference gate
    md_k, md_r = got['max_depth'].double().to(ref['ts'].device).reshape(n), ref['max_depth'].reshape(n)
    md_bad = (md_k - md_r).abs() > TOL['ts'][0] + TOL['ts'][1] * md_r.abs()
    md_bad = md_bad if rows is None else md_bad & rows
    sel = md_bad.nonzero()[:, 0]
    ts_k = got['ts'].double().to(sel.device).reshape(n, S)[sel]
    idx_k = (ts_k - got['max_depth'].double().to(sel.device).reshape(n)[sel, None]).abs().argmin(-1)
    sub = {'weights': ref['weights'][sel], 'deltas': ref['deltas'][sel], 'max_idx': ref['max_idx'][sel]}
    rep['max_idx'] = _idx_report(idx_k, sub, S) if sel.numel() else {'mismatch': 0, 'mismatch_not_tie': 0, 'mismatch_score_off': 0}
    g_vol, g_inv, mass = gref
    gs, gs_ref = grads['vol'][0].double().to(g_vol.device), g_vol[0]
    scale = float(gs_ref.abs().max())
    rep['grad_sdf'] = (float((gs - gs_ref).abs().max()) / (1e-3 * kappa * max(scale, 1.0)), float((gs - gs_ref).abs().max()))
    if g_vol.shape[0] > 1:
        gf, gf_ref = grads['vol'][1:].double().to(g_vol.device), g_vol[1:]
        scale = float(gf_ref.abs().max())
        rep['grad_feat'] = (float((gf - gf_ref).abs().max()) / (2e-4 * kappa * max(scale, 1.0)), float((gf - gf_ref).abs().max()))
    # d/d inv_s: like every gradient its relative tolerance scales with kappa; it also sums one signed term per sample
    # (fp32, tree + atomics; ~4e3 samples in the small test, ~5e5 here), each carrying the ~1e-7 absolute error of the
    # fast logistics through 1 - pa and 1 / (pa + 1e-5)^2, so the sum may also miss by 2^-13 of the terms' summed magnitude
    gi, gi_ref = float(grads['inv_s']), float(g_inv)
    rep['grad_inv_s'] = (abs(gi - gi_ref) / (2e-3 * kappa * max(1.0, abs(gi_ref)) + 2.0 ** -13 * mass), abs(gi - gi_ref))
    rep['inv_s_grad'] = [gi_ref, mass]
    return rep


def _passes(rep):
    ok = all(v[0] <= 1.0 for k, v in rep.items() if isinstance(v, tuple))
    return ok and rep['max_idx']['mismatch_not_tie'] == 0 and rep['max_idx']['mismatch_score_off'] == 0


def train_parity(got, grads, cot, vol64, mapping, o, d, nrm, aabb, inv_s, S, grid, jitter=None, color_dims=0,
                 bkgd_rand=None, tol=1e-4, geo_tol=5e-4, max_flip_frac=0.02, chunk=512):
    """got: kernel outputs (any device) in RenderTrainFunction names; grads: {'vol': [Cf,H,W,Z] kernel gradient of
    sum_k <got_k, cot_k>, 'inv_s': scalar}; cot: the cotangents the kernel backward ran with, zero on ``flip_rays`` rays;
    vol64 [Cf,H,W,Z] fp64; o, d, nrm fp64 flat rays (d unit); grid [n,S,3] the kernel's sample coordinates (probe).
    (b) is asserted on every ray with the tolerances of TOL times kappa (see A0); (c) as in the inference gate: every ray
    whose depth misses ``tol`` times kappa has a cell flip, and flip rays are at most ``max_flip_frac``.  The per-sample
    and gradient comparisons of (c) are reported: there the fp64 coordinates differ from the kernel's by rounding.
    Returns the report dict with ``ok``."""
    dev = vol64.device
    n = o.shape[0]
    g64, clip = sample_geometry(mapping, o, d, aabb, S, jitter)
    gk = grid.double().to(dev).reshape(n, S, 3)
    flip = flip_rays(gk, g64)
    for k in DIFF:
        if k in cot:
            assert not cot[k].to(dev)[flip].any(), 'cotangent %s is not zero on a flip ray' % k
    kw = dict(jitter=jitter, color_dims=color_dims, bkgd_rand=bkgd_rand, depth_clip=clip, chunk=chunk)
    same, *gsame = oracle_train(vol64, mapping, o, d, nrm, aabb, inv_s, S, cot, grid_override=gk, **kw)
    ind, *gind = oracle_train(vol64, mapping, o, d, nrm, aabb, inv_s, S, cot, **kw)
    rep = {'rays': n, 'inv_s': float(inv_s)}
    # deltas are differences of two fp32 edges over |dir|: 2 ulp of the farthest edge
    deltas_atol = 2.0 * float(torch.finfo(torch.float32).eps) * float(got['fars'].double().max())
    rep['geometry'] = {'max_abs_grid_units': float((gk - g64).abs().max()), 'tol': geo_tol, 'deltas_atol': deltas_atol}
    keep = ~flip
    e_same = alpha_arg_error(got, same, d, nrm)
    e_ind = alpha_arg_error(got, ind, d, nrm, rows=keep)
    k_same, k_ind = max(1.0, float(inv_s) * e_same / A0), max(1.0, float(inv_s) * e_ind / A0)
    rep['kappa'] = {'same_cells': k_same, 'independent': k_ind, 'alpha_arg_err_same': e_same, 'alpha_arg_err_ind': e_ind}
    rep['same_cells'] = _compare(got, same, grads, gsame, n, S, k_same, deltas_atol)
    rep['independent'] = _compare(got, ind, grads, gind, n, S, k_ind, deltas_atol, rows=keep)
    err = (got['depth'].double().to(dev).reshape(n) - ind['depth']).abs() / ind['depth'].abs().clamp_min(1e-6)
    over = err > tol * k_ind
    rep['independent'].update({'depth_max_rel': float(err.max()), 'rays_over_tol': int(over.sum()),
                               'rays_over_tol_without_cell_flip': int((over & ~flip).sum()), 'rays_with_cell_flip': int(flip.sum())})
    ok = (rep['geometry']['max_abs_grid_units'] <= geo_tol and _passes(rep['same_cells'])
          and rep['independent']['max_idx']['mismatch_not_tie'] == 0 and rep['independent']['max_idx']['mismatch_score_off'] == 0
          and rep['independent']['rays_over_tol_without_cell_flip'] == 0 and rep['independent']['rays_with_cell_flip'] <= max_flip_frac * n)
    rep['ok'] = bool(ok)
    return rep


def format_report(name, rep):
    f = lambda r: ' '.join('%s=%.2g(%.1e)' % (k, v[0], v[1]) for k, v in r.items() if isinstance(v, tuple))
    return ('%s: rays %d inv_s %.4g | d/d inv_s %.4g, term mass %.3g | geometry max %.1e | kappa same %.3g ind %.3g (alpha arg err %.1e / %.1e) | same cells [%s] '
            'max_idx %s | independent [%s] depth max rel %.1e, over tol %d (unattributed %d), flip rays %d, max_idx %s | ok=%s' % (
                name, rep['rays'], rep['inv_s'], *rep['same_cells']['inv_s_grad'], rep['geometry']['max_abs_grid_units'], rep['kappa']['same_cells'],
                rep['kappa']['independent'], rep['kappa']['alpha_arg_err_same'], rep['kappa']['alpha_arg_err_ind'],
                f(rep['same_cells']), rep['same_cells']['max_idx'], f(rep['independent']), rep['independent']['depth_max_rel'],
                rep['independent']['rays_over_tol'], rep['independent']['rays_over_tol_without_cell_flip'],
                rep['independent']['rays_with_cell_flip'], rep['independent']['max_idx'], rep['ok']))
