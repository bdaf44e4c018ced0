"""Oracle-side parity report for the render kernels (test infrastructure, see oracle/__init__.py).

Why three comparisons.  The reference's field is a trilinear interpolant (bev_nerf.py:99-117) whose ANALYTIC gradient
(``use_numerical_gradients=False``, config/nuscenes/nuscenes_depth.py:315) feeds the NeuS alpha; that gradient jumps
across cell faces.  A sample that lies within fp32 rounding of a face (|g - round(g)| ~ 1e-5 grid units) is therefore
assigned to one cell by any fp32 evaluation -- the reference's own included -- and possibly to the neighbour by an fp64
evaluation, and on a low-accumulation ray one such sample moves the expected depth by up to ~1e-2 relative (the fp32
ORACLE misses the fp64 oracle on such rays as well; scripts/parity_diag.py reports both).  So the gate separates the questions:

  (a) geometry   : the kernel's sample coordinates (probe output) equal the fp64 oracle's within rounding
                   (|dg| <= geo_tol grid units) -- a continuous quantity, no discontinuity involved;
  (b) same cells : fp64 oracle evaluated AT the kernel's coordinates (exactly representable in fp64) vs the kernel:
                   depth within ``tol`` relative (north-star 1e-4) on EVERY ray, acc / rgb / normals within abs tolerances,
                   max-depth index equal except provable near-ties -- this is "same function, same arithmetic";
  (c) independent: the plain fp64 oracle vs the kernel: every ray beyond ``tol`` must contain a sample whose cell differs
                   between the two evaluations (the mismatch is attributed, not waved through), those rays are counted and
                   bounded, and AbsRel (utils/metric_util.py:247-265) over all rays is reported.
"""
import torch

from . import render as orender
from .metric import cal_depth_metric_ref


def _rel(a, b):
    return (a - b).abs() / b.abs().clamp_min(1e-6)


def _idx_report(idx_k, ref, S):
    """max-depth index rule (neus_head.py:430-438): first maximum of w / clamp(delta, eps).  A mismatch is accepted only
    where the oracle's two best scores are a rounding-level tie (relative gap < 1e-5); ties are counted."""
    n = idx_k.numel()
    w, dl = ref['weights'].reshape(n, S), ref['deltas'].reshape(n, S)
    score = w / dl.clamp_min(torch.finfo(torch.float32).eps)
    top2 = score.topk(2, -1).values
    tie = (top2[:, 0] - top2[:, 1]) <= 1e-5 * top2[:, 0].abs().clamp_min(1e-300)
    ref_idx = ref['max_idx'].reshape(n)
    bad = idx_k.reshape(n) != ref_idx
    got = score.gather(1, idx_k.reshape(n, 1).long())[:, 0]
    near = (top2[:, 0] - got) <= 1e-4 * top2[:, 0].abs().clamp_min(1e-300)
    return {'equal_frac': float((~bad).float().mean()), 'mismatch': int(bad.sum()), 'mismatch_not_tie': int((bad & ~tie).sum()),
            'mismatch_score_off': int((bad & ~near).sum()), 'tie_rays': int(tie.sum())}


def render_parity(got, vol64, mapping, origin, direction, aabb, inv_s, S, color_dims=0, tol=1e-4, geo_tol=5e-4,
                  max_flip_frac=0.02, **kw):
    """got: kernel outputs on the CPU -- depth [n], acc [n], max_idx [n], grid [n,S,3] (probe) and optionally rgb [n,3],
    normal_vis [n,3]; vol64 [Cf,H,W,Z] fp64 decoded volume; origin [1,N,3] / direction [1,N,R,3] fp32 rays as the reference
    builds them.  Returns the report dict with ``ok``."""
    o64, d64 = origin.double(), direction.double()
    n = got['depth'].numel()
    gk = got['grid'].double().reshape(n, S, 3)
    ind = orender.head_render_ref(vol64, mapping, o64, d64, aabb, inv_s, S=S, color_dims=color_dims, **kw)
    same = orender.head_render_ref(vol64, mapping, o64, d64, aabb, inv_s, S=S, color_dims=color_dims, grid_override=gk, **kw)
    g64 = ind['grid'].reshape(n, S, 3)
    rep = {'rays': n, 'tolerance_rel': tol}
    # (a) geometry
    rep['geometry'] = {'max_abs_grid_units': float((gk - g64).abs().max()), 'tol': geo_tol}
    flip = (gk.floor() != g64.floor()).any(-1).any(-1)
    # (b) same cells
    dk = got['depth'].double().reshape(n)
    e_same = _rel(dk, same['depth'].reshape(n))
    b = {'depth_max_rel': float(e_same.max()), 'acc_max_abs': float((got['acc'].double().reshape(n) - same['acc'].reshape(n)).abs().max()),
         'max_idx': _idx_report(got['max_idx'], same, S)}
    if 'normal_vis' in got:
        b['normal_max_abs'] = float((got['normal_vis'].double().reshape(n, 3) - same['vis_normal'].reshape(n, 3)).abs().max())
    if color_dims and 'rgb' in got:
        b['rgb_max_abs'] = float((got['rgb'].double().reshape(n, 3) - same['rgb'].reshape(n, 3)).abs().max())
    rep['same_cells'] = b
    # (c) independent
    di = ind['depth'].reshape(n)
    e_ind = _rel(dk, di)
    over = e_ind > tol
    m = cal_depth_metric_ref(dk, di.clamp(1e-3, 80))
    acc64 = ind['acc'].reshape(n)
    rep['independent'] = {'depth_max_rel': float(e_ind.max()), 'rays_over_tol': int(over.sum()),
                          'rays_over_tol_without_cell_flip': int((over & ~flip).sum()), 'rays_with_cell_flip': int(flip.sum()),
                          'depth_max_rel_no_flip_rays': float(e_ind[~flip].max()) if (~flip).any() else 0.0,
                          'abs_rel': float(m['abs_rel']), 'rmse': float(m['rmse']), 'a1': float(m['a1']),
                          'acc_max_abs': float((got['acc'].double().reshape(n) - acc64).abs().max()),
                          'acc_min': float(acc64.min()), 'acc_median': float(acc64.median()),
                          'max_idx_equal_frac': float((got['max_idx'].reshape(n) == ind['max_idx'].reshape(n)).float().mean())}
    ok = (rep['geometry']['max_abs_grid_units'] <= geo_tol and b['depth_max_rel'] <= tol and b['acc_max_abs'] <= 2e-5
          and b['max_idx']['mismatch_not_tie'] == 0 and b['max_idx']['mismatch_score_off'] == 0
          and b.get('normal_max_abs', 0.0) <= 1e-4 and b.get('rgb_max_abs', 0.0) <= 1e-4
          and rep['independent']['rays_over_tol_without_cell_flip'] == 0
          and rep['independent']['rays_with_cell_flip'] <= max_flip_frac * n and rep['independent']['abs_rel'] <= 1e-5)
    rep['ok'] = bool(ok)
    return rep
