"""Training-form forward of NeuSHead (reference model/head/neus_head/neus_head.py:473-713): same output dict,
driven by the warp-per-ray training kernels (``so_render_train_forward/backward``)."""
import os
import torch

from . import ops


def chunk_cams(tensor, num_cams):
    """neus_head.py:716-721."""
    return [t.squeeze() for t in torch.chunk(tensor.reshape(num_cams, -1), num_cams, dim=0)]


def forward_train(head, representation, metas=None, jitter=None, bkgd_rand=None, uniform_shift=None, **kwargs):
    """uniform_shift: the [H*W*D, 3] lattice jitter in [0, 1) of get_uniform_sdf (default: drawn here).

    Ray-sharded training: with ``head.ray_shard = (rank, world)``, world > 1, this rank renders the rank-th contiguous slice
    (dist.ray_slice) of every camera's rays and ``outputs['ray_shard'] = (rank, world, R_full)`` tells MultiLoss to gather
    its inputs across the ranks.  Every rank must see the same frame and the same random numbers: give every rank the same
    training frames (a distributed sampler that hands each rank its own frames must be built with one replica) and seed
    torch AND numpy identically on all ranks (the reference's train.py seeds them; INTEGRATION.md lists what else it needs
    for a sharded run).  The cellular ray grid comes from numpy (RaySampler.draw); the stratified
    jitter and the random background are drawn for all rays and sliced; the uniform_sdf lattice shift and the encoder's
    dropout masks are then drawn identically.  An explicit ``jitter`` / ``bkgd_rand`` is this rank's slice."""
    f = head.model.field
    hw, zh, wz = representation
    assert hw.shape[0] == 1, 'only support bs = 1 currently'
    l1, l2 = f.density_net[1], f.density_net[3]
    vol_sdf, vol_feat = ops.TPVDecodeFunction.apply(hw[0], zh[0], wz[0], l1.weight, l1.bias, l2.weight, l2.bias, f.desc)
    vol_feat = vol_feat if f.desc.n_feat else None
    f.vol_sdf, f.vol_feat = vol_sdf.detach(), (vol_feat.detach() if vol_feat is not None else None)
    f.vol_sdf_live, f.vol_feat_live = vol_sdf, vol_feat           # autograd-connected views for get_uniform_sdf
    dev = vol_sdf.device

    sampler = head._sampler()
    grid = sampler.draw()
    rays = sampler.table(grid)
    r_full = rays.shape[0]
    shard = getattr(head, 'ray_shard', None)
    sharded = shard is not None and shard[1] > 1
    if sharded:
        # ray-sharded training (BASELINE configs[4]): rank r renders the r-th contiguous slice of EVERY camera's pixel rays, so the
        # per-camera output lists the losses consume keep their structure (fewer rays per camera); MultiLoss gathers the loss
        # inputs across the ranks (outputs['ray_shard'])
        from .dist import ray_slice
        b, c = ray_slice(r_full, shard[1], shard[0])
        rays, grid = rays[b:b + c].contiguous(), None
    M = head.img2lidar.matrices(metas, dev)
    bs, num_cams = M.shape[:2]
    assert bs == 1, 'only support bs = 1 currently'
    num_rays = rays.shape[0]
    total = num_cams * num_rays
    S = head.num_samples
    training = head.training

    def draw(k):
        """torch.rand for every camera's rays; a sharded rank draws the FULL set and keeps its slice, so every rank consumes
        the torch RNG identically and its rays get the numbers the unsharded step gives them"""
        if not sharded:
            return torch.rand(total, k, device=dev)
        return torch.rand(num_cams, r_full, k, device=dev)[:, b:b + c].reshape(total, k)
    if jitter is None and training:                       # perturb=True: stratified jitter (upstream UniformSampler)
        jitter = draw(S + 1)
    has_rgb = f.color_dims >= 3
    if bkgd_rand is None and head.render_bkgd == 'random' and has_rgb:
        bkgd_rand = draw(3)
    inv_s = f.deviation_network.get_variance()
    params = ops.make_render_params(head.aabb, S, float(inv_s), near_plane=head.near_plane, training=training,
                                    cos_anneal=head.cos_anneal_ratio, anchor_mid=head.sample_anchor == 'mid', sh_act=f.sh_act,
                                    bkgd=head.render_bkgd)
    rd = ops.make_ray_desc(num_cams, grid=grid, n_pix=num_rays)
    want = ['depth', 'acc', 'fars', 'weights', 'ts', 'deltas', 'eik_grad']
    want += ['rgb'] if has_rgb else []
    want += ['sem'] if head.return_sem else []
    want += ['max_depth'] if head.return_max_depth else []
    want += ['sample_sdf'] if head.return_sample_sdf else []
    cfg = dict(desc=f.desc, cam_mats=M[0].contiguous(), rays=rd, params=params, pix=None if grid is not None else rays.contiguous(),
               jitter=jitter, bkgd_rand=bkgd_rand, want=want)
    res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vol_sdf, vol_feat, inv_s, cfg)))

    shp = (bs, num_cams, num_rays)
    depth, acc, fars = res['depth'].reshape(shp), res['acc'].reshape(shp), res['fars'].reshape(shp)
    rgb = res['rgb'].reshape(*shp, 3) if has_rgb else depth.new_empty(*shp, 0)
    weights = res['weights'].reshape(*shp, S, 1)
    ts = res['ts'].reshape(total, S, 1)
    deltas = res['deltas'].reshape(total, S, 1)
    # img2lidar outputs kept for API parity (neus_head.py:674-676)
    origin, direction = head.img2lidar(metas, rays)
    origin = origin.unsqueeze(2).repeat(1, 1, num_rays, 1).flatten(0, 2)
    direction = direction.flatten(0, 2)
    direction_norm = torch.norm(direction, dim=-1, keepdim=True)
    direction = direction / direction_norm

    uniform_sdf = None
    if head.return_uniform_sdf:
        uniform_sdf = _uniform_sdf_train(head, dev, uniform_shift)
    weights_for_cams = chunk_cams(weights, num_cams)
    ts_for_cams = chunk_cams(ts, num_cams)
    deltas_for_cams = chunk_cams(deltas, num_cams)
    ray_idx = [torch.arange(num_rays, device=dev).unsqueeze(-1).repeat(1, S).flatten()] * num_cams
    sem = res['sem'].reshape(*shp, -1) if head.return_sem else None
    max_depth = res['max_depth'].reshape(shp) if head.return_max_depth else None
    sample_sdf_for_cams = chunk_cams(res['sample_sdf'].reshape(*shp, S), num_cams) if head.return_sample_sdf else None

    if head.two_split and head.img2lidar.two_split:      # neus_head.py:647-665
        half = num_cams // 2
        depth, acc, fars = depth[:, :half], acc[:, :half], fars[:, :half]
        rgb = rgb[:, half:]
        ray_idx, weights_for_cams = ray_idx[:half], weights_for_cams[:half]
        ts_for_cams, deltas_for_cams = ts_for_cams[:half], deltas_for_cams[:half]
        if max_depth is not None:
            max_depth = max_depth[:, :half]
        if sample_sdf_for_cams is not None:
            sample_sdf_for_cams = sample_sdf_for_cams[:half]
        if sem is not None:
            sem = sem[:, half:]

    outputs = {'ms_depths': [depth], 'ms_colors': [rgb], 'ms_accs': [acc], 'ms_fars': [fars], 'ms_rays': rays,
               'origin': origin, 'direction': direction, 'direction_norm': direction_norm, 'ray_indices': ray_idx,
               'weights': weights_for_cams, 'ts': ts_for_cams, 'deltas': deltas_for_cams,
               'eik_grad': res['eik_grad'].reshape(total, S, 3), 'uniform_sdf': uniform_sdf, 'inv_s': inv_s}
    if head.return_max_depth:
        outputs['ms_max_depths'] = [max_depth]
    if head.return_second_grad:
        # opt-in DECLARED ASSUMPTION (so_field_second_grad): row sums of the Hessian of the trilinear field at the samples
        t_len = (ts if head.sample_anchor == 'mid' else ts - 0.5 * deltas) * direction_norm[:, None, :]      # ray length at the query point
        pos = (origin[:, None, :] + direction[:, None, :] * t_len).detach().reshape(-1, 3).contiguous()
        outputs['second_grad'] = ops.FieldSecondGradFunction.apply(vol_sdf, f.desc, pos).reshape(total, S, 3)
    if head.return_surface_sdf:
        raise NotImplementedError('return_surface_sdf needs the fork\'s `surface_points` definition (unrecoverable, DESIGN.md)')
    if head.return_sample_sdf:
        outputs['sample_sdf'] = sample_sdf_for_cams
    if head.return_sem:
        outputs['sem'] = [sem]
    if sharded:
        outputs['ray_shard'] = (shard[0], shard[1], r_full)
    return outputs


def uniform_lattice_train(head, dev):
    """The [H, W, D, 3] metre lattice of get_uniform_sdf (neus_head.py:266-277) on ``dev``."""
    a, r = head.aabb, head.resolution
    xs = torch.linspace(a[0], a[3], int((a[3] - a[0]) / r), device=dev)
    ys = torch.linspace(a[1], a[4], int((a[4] - a[1]) / r), device=dev)
    zs = torch.linspace(a[2], a[5], int((a[5] - a[2]) / r), device=dev)
    W, H, D = len(xs), len(ys), len(zs)
    return torch.stack([xs[None, :, None].expand(H, W, D), ys[:, None, None].expand(H, W, D),
                        zs[None, None, :].expand(H, W, D)], dim=-1)


def _uniform_sdf_train(head, dev, shift=None):
    """get_uniform_sdf(aabb, resolution, shift=True) with gradients to the volume (neus_head.py:533-538)."""
    f = head.model.field
    lat = uniform_lattice_train(head, dev)
    H, W, D = lat.shape[:3]
    xyz = lat.flatten(0, 2)
    if shift is None:
        shift = torch.rand_like(xyz)
    assert shift.shape == xyz.shape, 'uniform_shift must be [H*W*D, 3]'
    xyz = (xyz + shift * head.resolution).contiguous()
    s, _, _ = ops.FieldQueryFunction.apply(f.vol_sdf_live, f.vol_feat_live, f.desc, xyz, False, False)
    return s.reshape(H, W, D)
