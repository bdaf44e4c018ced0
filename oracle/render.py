"""Oracle: SDF volume-render head (test infrastructure, see oracle/__init__.py).

PARITY UNPINNED.  The arithmetic of this path lives in the un-vendored, un-pinned
``huang-yh/sdfstudio`` fork (reference model/head/neus_head/neus_head.py:2-6,129-197).
What is restated here, and from where:

* TPV -> dense decoded volume: the in-repo analogue model/head/nerfacc_head/bev_nerf.py:62-95
  (``tpv=True`` branch: broadcast-sum of the three planes, Softplus/Linear MLP).
* field query = ``meter2grid(x, normalize=True)`` then 3-D ``F.grid_sample(bilinear,
  align_corners=True, zeros padding)`` with the (d, w, h) axis order: bev_nerf.py:99-117 and
  the head's own use at neus_head.py:612-619.  Channel layout h = [sdf, rgb(3), sem...]:
  neus_head.py:284-288.  Colour = SH degree-0 ``relu(C0*f + 0.5)``: sh_render.py:84-94.
* collider / sampler / NeuS alpha / compositing / renderers: upstream sdfstudio semantics
  (AABB box collider, uniform 'spaced' sampler with optional stratified jitter, NeuS
  logistic-CDF alpha with learned inv_s, ``T = cumprod(1 - a + 1e-7)`` exclusive,
  expected-depth renderer with its batch-wide clip, depth / directions_norm), as named
  by the reference's constructor arguments neus_head.py:129-197 -- DECLARED ASSUMPTION.
  SDF spatial gradient = autograd of the trilinear interpolant w.r.t. the sample position
  (``use_numerical_gradients=False``, config/nuscenes/nuscenes_depth.py:315).
* post-processing (ts / deltas / max-depth argmax / uniform lattice): neus_head.py:265-293,
  366-374, 430-438, 571-587 -- in-repo, restated exactly.
"""
import math
import torch
import torch.nn.functional as F

C0 = 0.28209479177387814  # sh_render.py:4


def tpv_decode_ref(tpv_hw, tpv_zh, tpv_wz, sizes, w1, b1, w2, b2, h_chunk=16):
    """bev_nerf.py:81-95 with density_layers=2 (``Softplus, Linear(C,C), Softplus, Linear(C,Cf)``).

    tpv_hw [H*W, C], tpv_zh [Z*H, C], tpv_wz [W*Z, C]  ->  decoded volume [Cf, H, W, Z].
    Chunked over h only to bound the [h,W,Z,C] intermediate (the reference materialises it whole)."""
    H, W, Z = sizes
    C = tpv_hw.shape[-1]
    hw = tpv_hw.reshape(H, W, 1, C)
    zh = tpv_zh.reshape(Z, H, 1, C).permute(1, 2, 0, 3)  # H,1,Z,C
    wz = tpv_wz.reshape(W, Z, 1, C).permute(2, 0, 1, 3)  # 1,W,Z,C
    out = []
    for h0 in range(0, H, h_chunk):
        f = hw[h0:h0 + h_chunk] + zh[h0:h0 + h_chunk] + wz
        f = F.linear(F.softplus(f), w1, b1)
        f = F.linear(F.softplus(f), w2, b2)
        out.append(f)
    return torch.cat(out, 0).permute(3, 0, 1, 2).contiguous()


def field_query_ref(vol, mapping, x, with_grad=True):
    """vol [Cf,H,W,Z]; x [N,3] metres -> (h [N,Cf], grad_sdf [N,3] or None).  bev_nerf.py:155-170."""
    x = x.detach().to(vol.dtype).clone().requires_grad_(with_grad)
    with torch.enable_grad():
        g = mapping.meter2grid(x, True) * 2 - 1
        samp = F.grid_sample(vol[None], g.reshape(1, -1, 1, 1, 3)[..., [2, 1, 0]], mode='bilinear',
                             align_corners=True)  # 1,Cf,N,1,1
        h = samp[0, :, :, 0, 0].t()
        grad = None
        if with_grad:
            grad = torch.autograd.grad(h[:, 0].sum(), x)[0]
    return h.detach(), grad


def field_query_manual(vol, mapping, x, grid_override=None):
    """Same function as ``field_query_ref`` written as explicit 8-corner gathers so that BOTH outputs (values and
    the analytic position-gradient) are differentiable w.r.t. ``vol`` -- PyTorch has no double backward for
    ``grid_sampler_3d`` (the fork vendors ``cuda_gridsample_grad2`` for that, docs/installation.md:30).  Used by the
    training-parity tests; checked against ``field_query_ref`` in tests/test_oracle_selfcheck.py."""
    Cf, H, W, Z = vol.shape
    x = x.to(vol.dtype)
    # grid_override [N,3] (h, w, d): evaluate the interpolant at THESE grid coordinates (e.g. the fp32 coordinates a kernel
    # used, exactly representable in fp64) while the metre->grid slopes still come from x -- separates "same function"
    # from "same cell" when a sample sits within rounding of a cell face (the analytic gradient jumps there)
    g = mapping.meter2grid(x, False) if grid_override is None else grid_override.to(vol.dtype)
    gh, gw, gd = g[:, 0], g[:, 1], g[:, 2]
    h0, w0, z0 = gh.floor(), gw.floor(), gd.floor()
    fh, fw, fz = gh - h0, gw - w0, gd - z0
    h0, w0, z0 = h0.long(), w0.long(), z0.long()
    val = vol.new_zeros(x.shape[0], Cf)
    dgh = vol.new_zeros(x.shape[0])
    dgw = vol.new_zeros(x.shape[0])
    dgd = vol.new_zeros(x.shape[0])
    for dh in (0, 1):
        for dw in (0, 1):
            for dz in (0, 1):
                hh, ww, zz = h0 + dh, w0 + dw, z0 + dz
                ok = (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W) & (zz >= 0) & (zz < Z)
                v = vol[:, hh.clamp(0, H - 1), ww.clamp(0, W - 1), zz.clamp(0, Z - 1)].t() * ok[:, None].to(vol.dtype)
                wh = fh if dh else 1 - fh
                w_w = fw if dw else 1 - fw
                wz = fz if dz else 1 - fz
                val = val + (wh * w_w * wz)[:, None] * v
                dgh = dgh + (1.0 if dh else -1.0) * w_w * wz * v[:, 0]
                dgw = dgw + wh * (1.0 if dw else -1.0) * wz * v[:, 0]
                dgd = dgd + wh * w_w * (1.0 if dz else -1.0) * v[:, 0]
    # chain rule through the per-axis piecewise-linear metre->grid map
    xr = x.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        gg = mapping.meter2grid(xr, False)
        slopes = torch.autograd.grad(gg.sum(), xr)[0]          # d(grid of own axis)/d(metre): (kw, kh, kd) in x,y,z order
    grad = torch.stack([dgw * slopes[:, 0], dgh * slopes[:, 1], dgd * slopes[:, 2]], -1)
    return val, grad


def aabb_near_far(o, d, aabb, near_plane, training):
    """upstream AABBBoxCollider: slab test with 1/(d + 1e-6); near clamped to near_plane when
    training else 0; far >= near + 1e-6."""
    inv = 1.0 / (d + 1e-6)
    lo = torch.as_tensor(aabb[:3], dtype=o.dtype, device=o.device)
    hi = torch.as_tensor(aabb[3:], dtype=o.dtype, device=o.device)
    t1 = (lo - o) * inv
    t2 = (hi - o) * inv
    nears = torch.minimum(t1, t2).max(-1).values
    fars = torch.maximum(t1, t2).min(-1).values
    nears = nears.clamp(min=near_plane if training else 0.0)
    fars = torch.maximum(fars, nears + 1e-6)
    return nears, fars


def uniform_bins(nears, fars, S, jitter=None):
    """upstream UniformSampler: S bins, edges = near + (far-near)*linspace(0,1,S+1); stratified
    jitter (training, ``perturb=True``) re-draws each edge inside its half-cell given
    ``jitter`` in [0,1) of shape [R, S+1]."""
    bins = torch.linspace(0.0, 1.0, S + 1, dtype=nears.dtype, device=nears.device)[None]
    if jitter is not None:
        ctr = (bins[..., 1:] + bins[..., :-1]) / 2.0
        upper = torch.cat([ctr, bins[..., -1:]], -1)
        lower = torch.cat([bins[..., :1], ctr], -1)
        bins = lower + (upper - lower) * jitter
    e = bins * fars[:, None] + (1 - bins) * nears[:, None]
    return e[:, :-1], e[:, 1:]


def neus_render_chunk(vol, mapping, o, d, dnorm, aabb, inv_s, S=256, near_plane=0.0, training=False,
                      jitter=None, cos_anneal=1.0, color_dims=0, sh_act='relu', bkgd='white',
                      bkgd_rand=None, anchor='mid', differentiable=False, grid_override=None, depth_clip=None):
    """One ``self.model(ray_bundle)`` call of the reference (neus_head.py:353/394/531) for a chunk
    of rays o,d [R,3] (d unit), dnorm [R,1].  Returns the dict the head consumes.  ``depth_clip`` = (lo, hi): the
    expected-depth clip bounds of the whole batch when this call renders only a part of it (default: this chunk's)."""
    R = o.shape[0]
    nears, fars = aabb_near_far(o, d, aabb, near_plane, training)
    starts, ends = uniform_bins(nears, fars, S, jitter)
    mids = (starts + ends) / 2
    deltas = ends - starts
    tq = mids if anchor == 'mid' else starts
    x = o[:, None, :] + d[:, None, :] * tq[..., None]
    grid = mapping.meter2grid(x.detach(), False)               # [R,S,3] (h, w, d) unnormalised grid coordinates of the samples
    if grid_override is not None:
        h, grad = field_query_manual(vol, mapping, x.reshape(-1, 3), grid_override.reshape(-1, 3))
    elif differentiable:
        h, grad = field_query_manual(vol, mapping, x.reshape(-1, 3))
    else:
        h, grad = field_query_ref(vol, mapping, x.reshape(-1, 3))
    h = h.reshape(R, S, -1)
    grad = grad.reshape(R, S, 3)
    sdf = h[..., 0]
    # NeuS alpha (upstream SDFField.get_alpha)
    true_cos = (d[:, None, :] * grad).sum(-1)
    iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal) + F.relu(-true_cos) * cos_anneal)
    est_next = sdf + iter_cos * deltas * 0.5
    est_prev = sdf - iter_cos * deltas * 0.5
    prev_cdf = torch.sigmoid(est_prev * inv_s)
    next_cdf = torch.sigmoid(est_next * inv_s)
    alpha = ((prev_cdf - next_cdf + 1e-5) / (prev_cdf + 1e-5)).clip(0.0, 1.0)
    trans = torch.cumprod(torch.cat([torch.ones(R, 1, dtype=alpha.dtype, device=alpha.device), 1.0 - alpha + 1e-7], 1), 1)
    weights = alpha * trans[:, :-1]
    acc = weights.sum(-1)
    # expected-depth renderer incl. its chunk-wide clip, then ray-length -> camera-z units
    depth = (weights * mids).sum(-1) / (acc + 1e-10)
    depth = depth.clip(*(depth_clip if depth_clip is not None else (mids.min(), mids.max())))
    depth = depth / dnorm[:, 0]
    normals = F.normalize(grad, p=2, dim=-1)
    normal = (weights[..., None] * normals).sum(-2)
    out = dict(depth=depth, accumulation=acc, weights=weights, starts=starts, ends=ends, sdf=sdf,
               eik_grad=grad, normal=normal, normal_vis=(normal + 1.0) / 2.0, nears=nears,
               fars=fars / dnorm[:, 0], alpha=alpha, grid=grid)
    if color_dims > 0:
        raw = h[..., 1:4] * C0  # SH degree 0 (sh_render.py:84-94)
        rgb_s = torch.relu(raw + 0.5) if sh_act == 'relu' else torch.sigmoid(raw)
        rgb = (weights[..., None] * rgb_s).sum(-2)
        if bkgd == 'white':
            bg = torch.ones(3, device=o.device)
        elif bkgd == 'black':
            bg = torch.zeros(3, device=o.device)
        elif bkgd == 'random':
            bg = bkgd_rand
        else:
            raise NotImplementedError(bkgd)
        rgb = rgb + bg * (1.0 - acc[:, None])
        if not training:
            rgb = rgb.clamp(0.0, 1.0)
        out['rgb'] = rgb
        if h.shape[-1] > 4:
            out['sem'] = (weights[..., None] * torch.softmax(h[..., 4:], -1)).sum(-2)
    else:
        out['rgb'] = torch.empty(R, 0, device=o.device)  # bev_nerf.py:145-146: no colour channels decoded
    return out


def max_depth_ref(weights, ts, deltas):
    """neus_head.py:430-438 / 579-587.  weights, ts, deltas [..., S] -> (max_depth, index int64).  The reference renders in
    fp32, so a sample is dropped below fp32's eps whatever dtype the oracle runs in: a ray that misses the ROI has
    zero-length samples (far - near = 1e-6), all dropped, and takes index 0."""
    eps = torch.finfo(torch.float32).eps
    w = weights.clone()
    w[deltas < eps] = 0.
    idx = (w / deltas.clamp_min(eps)).argmax(-1, keepdim=True)
    return torch.gather(ts, -1, idx).squeeze(-1), idx.squeeze(-1)


def head_render_ref(vol, mapping, origin, direction, aabb, inv_s, batch=0, max_depth_on_cpu=False, grid_override=None, **kw):
    """NeuSHead.render (neus_head.py:308-471) after ray generation: origin [1,N,3], direction
    [1,N,R,3] un-normalised.  Serial chunk loop with ``torch.chunk`` sizes when batch > 0.  ``bkgd_rand`` (bkgd='random')
    holds one row per ray, [N*R, 3] in the flat (cam, ray) order, and is chunked with the rays."""
    from .rays import flatten_rays, num_chunks
    bs, n_cam, n_ray = direction.shape[:3]
    o, d, nrm = flatten_rays(origin, direction)
    n = num_chunks(o.shape[0], batch)
    go = [None] * n if grid_override is None else torch.chunk(grid_override.reshape(o.shape[0], -1, 3), n)
    bk = kw.pop('bkgd_rand', None)
    bk = [None] * n if bk is None else torch.chunk(bk.reshape(o.shape[0], 3), n)
    outs = [neus_render_chunk(vol, mapping, oc, dc, nc, aabb, inv_s, grid_override=gc, bkgd_rand=bc, **kw)
            for oc, dc, nc, gc, bc in zip(torch.chunk(o, n), torch.chunk(d, n), torch.chunk(nrm, n), go, bk)]
    cat = lambda k: torch.cat([c[k] for c in outs])
    weights = cat('weights')
    ts = (cat('starts') + cat('ends')) / 2 / nrm
    deltas = (cat('ends') - cat('starts')) / nrm
    if max_depth_on_cpu:        # neus_head.py:430-438 moves weights / deltas / ts to the host for this step
        max_depth, max_idx = max_depth_ref(weights.cpu(), ts.cpu(), deltas.cpu())
        max_depth, max_idx = max_depth.to(weights.device), max_idx.to(weights.device)
    else:
        max_depth, max_idx = max_depth_ref(weights, ts, deltas)
    shp = (bs, n_cam, n_ray)
    return dict(depth=cat('depth').reshape(shp), acc=cat('accumulation').reshape(shp),
                rgb=cat('rgb').reshape(*shp, -1), vis_normal=cat('normal_vis').reshape(*shp, 3),
                max_depth=max_depth.reshape(shp), max_idx=max_idx.reshape(shp),
                weights=weights.reshape(*shp, -1), ts=ts.reshape(*shp, -1), deltas=deltas.reshape(*shp, -1),
                sdf=cat('sdf').reshape(*shp, -1), eik_grad=cat('eik_grad').reshape(*shp, -1, 3),
                fars=cat('fars').reshape(shp), grid=cat('grid').reshape(*shp, -1, 3),
                sem=cat('sem').reshape(*shp, -1) if 'sem' in outs[0] else None)


def uniform_lattice(aabb, resolution):
    """neus_head.py:266-277: inclusive-endpoint linspace lattice, [H(y), W(x), D(z), 3] metres."""
    xs = torch.linspace(aabb[0], aabb[3], int((aabb[3] - aabb[0]) / resolution))
    ys = torch.linspace(aabb[1], aabb[4], int((aabb[4] - aabb[1]) / resolution))
    zs = torch.linspace(aabb[2], aabb[5], int((aabb[5] - aabb[2]) / resolution))
    W, H, D = len(xs), len(ys), len(zs)
    return torch.stack([xs[None, :, None].expand(H, W, D), ys[:, None, None].expand(H, W, D),
                        zs[None, None, :].expand(H, W, D)], -1)


def uniform_sdf_ref(vol, mapping, aabb, resolution, shift=None):
    """neus_head.py:265-293 (get_uniform_sdf): sdf [H,W,D] (+ sem logits h[...,4:] when decoded)."""
    xyz = uniform_lattice(aabb, resolution)
    if shift is not None:
        xyz = xyz + shift * resolution
    h, _ = field_query_ref(vol, mapping, xyz.reshape(-1, 3), with_grad=False)
    H, W, D = xyz.shape[:3]
    sdf = h[:, 0].reshape(H, W, D)
    sem = h[:, 4:].reshape(H, W, D, -1) if h.shape[1] > 4 else None
    return sdf, sem, xyz
