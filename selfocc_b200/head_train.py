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
    dropout masks are then drawn identically.  An explicit ``jitter`` / ``bkgd_rand`` is this rank's slice.

    Fused objective (``head.fused_objective``, set by loss.fuse_objective; training mode only): the render computes the
    reprojection statistics and the eikonal mean itself (RenderTrainObjectiveFunction) and the outputs carry
    ``reproj_stats`` [num_cams, R, 6 * sets], ``reproj_colours`` [num_cams, R, 9] and ``eikonal_mean`` (0-d) in place of
    ``weights``, ``ts``, ``deltas`` and ``eik_grad``.  The reprojection term's images arrive as the model kwargs
    ``curr_imgs`` / ``prev_imgs`` / ``next_imgs`` ([1, num_cams, 3, H, W]) and its matrices as metas' img2prevImg /
    img2nextImg.  With ``second_grad`` fused as well (fuse_objective(..., second_grad=True)) the render also takes the
    second-grad mean at its own sample points and the outputs carry ``second_grad_mean`` (0-d) in place of ``second_grad``;
    no per-sample tensor is then requested from the render.

    Decode-sharded training (``head.decode_shard = (rank, world)``, world > 1; training mode with grad enabled): see
    decode_train.  The gathered volume feeds the render, ``uniform_sdf``, ``second_grad`` and the fused objective alike."""
    f = head.model.field
    vol_sdf, vol_feat = decode_train(head, representation)
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
    fused = getattr(head, 'fused_objective', None) if training else None
    fused_sg = fused is not None and fused.get('second_grad', False)
    if fused is None:
        want = ['depth', 'acc', 'fars', 'weights', 'ts', 'deltas', 'eik_grad']
    else:                                                  # sample positions only for an unfused second-grad query
        want = ['depth', 'acc', 'fars'] + (['ts', 'deltas'] if head.return_second_grad and not fused_sg else [])
    want += ['rgb'] if has_rgb else []
    want += ['sem'] if head.return_sem else []
    want += ['max_depth'] if head.return_max_depth else []
    want += ['sample_sdf'] if head.return_sample_sdf else []
    cfg = dict(desc=f.desc, cam_mats=M[0].contiguous(), rays=rd, params=params, pix=None if grid is not None else rays.contiguous(),
               jitter=jitter, bkgd_rand=bkgd_rand, want=want)
    if fused is None:
        res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vol_sdf, vol_feat, inv_s, cfg)))
    else:
        cfg['objective'] = _objective(fused, kwargs, metas, rays, num_cams, dev)
        res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER, ops.RenderTrainObjectiveFunction.apply(vol_sdf, vol_feat, inv_s, cfg)))

    shp = (bs, num_cams, num_rays)
    depth, acc, fars = res['depth'].reshape(shp), res['acc'].reshape(shp), res['fars'].reshape(shp)
    rgb = res['rgb'].reshape(*shp, 3) if has_rgb else depth.new_empty(*shp, 0)
    if 'ts' in want:
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
    if fused is None:
        weights_for_cams = chunk_cams(res['weights'].reshape(*shp, S, 1), num_cams)
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
               'origin': origin, 'direction': direction, 'direction_norm': direction_norm, 'ray_indices': ray_idx}
    if fused is None:
        outputs.update(weights=weights_for_cams, ts=ts_for_cams, deltas=deltas_for_cams, eik_grad=res['eik_grad'].reshape(total, S, 3))
    else:
        if fused['mode'] is not None:
            outputs.update(reproj_stats=res['reproj_stats'].reshape(num_cams, num_rays, -1),
                           reproj_colours=res['reproj_colours'].reshape(num_cams, num_rays, 9))
        if fused['eikonal']:
            outputs['eikonal_mean'] = res['eikonal_mean']
        if fused_sg:
            outputs['second_grad_mean'] = res['second_grad_mean']
    outputs.update(uniform_sdf=uniform_sdf, inv_s=inv_s)
    if head.return_max_depth:
        outputs['ms_max_depths'] = [max_depth]
    if head.return_second_grad and not fused_sg:
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


def decode_train(head, representation):
    """The training form of the decode -> (vol_sdf, vol_feat; an empty tensor when no features are decoded).

    With ``head.decode_shard = (rank, world)``, world > 1, in training mode with grad enabled, this rank decodes only its
    slab of the volume's h rows (dist.volume_slab: H < world is refused) and dist.all_gather_volume assembles the full volume
    on every rank over ``head.decode_shard_group`` (``head.decode_shard_collectives``: optional (collective,
    reduce_scatter) hooks in its place): one all_gather forward, one reduce-scatter of the volume gradient backward.  The
    decode's backward then runs over the slab's rows only.  Both fields (tpv True / False) shard the same way.

    Gradient rule (DESIGN.md section 6): a rank's gradient w.r.t. the full volume is partial and scaled by world under
    ``head.ray_shard``, full and unscaled for the replicated terms (uniform_sdf, second_grad, any term of a step without ray
    sharding); either way the sum over the ranks is world x the full gradient.  The reduce-scatter hands rank r world x the
    full gradient on its slab, so its plane and MLP-weight gradients are world x the slab's share, and their sum over the
    ranks is world x the full gradient: DistributedDataParallel's mean is exact.  Eval and no_grad ignore the switch
    (inference shards its decode with dist.decode_sharded)."""
    f = head.model.field
    shard = getattr(head, 'decode_shard', None)
    if shard is None or shard[1] <= 1 or not (head.training and torch.is_grad_enabled()):
        return f.decode(representation, train=True)
    from .dist import all_gather_volume, volume_slab
    rank, world = shard
    rows = volume_slab(f.desc.H, rank, world)
    vs, vf = f.decode(representation, train=True, rows=rows)
    hooks = getattr(head, 'decode_shard_collectives', None) or (None, None)
    vs, vf = all_gather_volume(vs, vf if f.desc.n_feat else None, f.desc.H, rank, world, *hooks,
                               group=getattr(head, 'decode_shard_group', None))
    return vs, (vf if vf is not None else vs.new_empty(0))


def _objective(fused, kwargs, metas, rays, num_cams, dev):
    """RenderTrainObjectiveFunction's cfg['objective'] from head.fused_objective: the reprojection term's loss pixels (the
    rays), matrices (metas, as the loss reads them) and images (the model kwargs), and whether the eikonal and second-grad
    means are on."""
    ob = dict(mode=fused['mode'], eikonal=fused['eikonal'], second_grad=fused.get('second_grad', False))
    if fused['mode'] is None:
        return ob
    from .loss import _mats
    keys = ('curr_imgs', 'prev_imgs', 'next_imgs')
    missing = [k for k in keys if kwargs.get(k) is None]
    if missing:
        raise ValueError('the fused objective renders the reprojection statistics from the images: call the model with '
                         'curr_imgs=, prev_imgs=, next_imgs= (missing %s)' % missing)
    ob.update(pix=rays.detach().float().contiguous(), img2prev=_mats(metas, 'img2prevImg', num_cams, dev),
              img2next=_mats(metas, 'img2nextImg', num_cams, dev),
              images=tuple(kwargs[k][0, :num_cams].float().contiguous() for k in keys), img_size=fused['img_size'])
    return ob


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
