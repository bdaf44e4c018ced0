"""Multi-GPU plumbing for the render path (SURVEY.md 8e): rays are independent given the decoded
volume, so the flat (cam, ray) order of neus_head.py:324-325 is split into contiguous per-rank slices
(the same split ``torch.chunk`` produces) and the rendered maps are put back together with ONE
all_gather.  Ray-sharded TRAINING slices every camera's rays instead (head.ray_shard) and gathers the loss
inputs per camera, differentiably (all_gather_ray_payload).  Backend-agnostic (``nccl`` on the GPUs, ``gloo`` in
the CPU tests)."""
import math

import torch
import torch.distributed as dist

from . import ops


def ray_slice(total, world_size, rank):
    """(begin, count) of this rank's contiguous slice; identical to torch.chunk(arange(total), world_size)."""
    per = -(-total // world_size)
    begin = min(rank * per, total)
    return begin, max(0, min(per, total - begin))


def all_gather_rays(local, total, group=None):
    """local [count, ...] of this rank -> [total, ...] in flat ray order on every rank.  One collective:
    slices are padded to the common per-rank length so a single all_gather_into_tensor suffices."""
    if not dist.is_available() or not dist.is_initialized():
        return local
    world = dist.get_world_size(group)
    per = -(-total // world)
    tail = local.shape[1:]
    buf = local
    if local.shape[0] != per:
        buf = local.new_zeros((per,) + tuple(tail))
        buf[:local.shape[0]] = local
    out = local.new_empty((world * per,) + tuple(tail))
    try:
        dist.all_gather_into_tensor(out, buf.contiguous(), group=group)
    except (RuntimeError, NotImplementedError):        # older gloo builds: list form, still one collective
        parts = [torch.empty_like(buf) for _ in range(world)]
        dist.all_gather(parts, buf.contiguous(), group=group)
        out = torch.cat(parts, 0)
    return out[:total]


def pack_planar(tensors, totals, world, dtype=None):
    """This rank's payload -> the 1-D buffer one all_gather_into_tensor exchanges.  tensors[i] is [L, count_i, k] (L rows of
    slices, e.g. one per camera); its slice is padded to ceil(totals[i] / world) along dim 1.  The buffer is PLANAR (tensor
    after tensor -- contiguous copies; an interleaved [count, sum k] pack would cost a strided write of every column)."""
    sizes = [t.shape[0] * -(-n // world) * t.shape[2] for t, n in zip(tensors, totals)]
    buf = tensors[0].new_zeros(sum(sizes), dtype=dtype)
    off = 0
    for t, n, size in zip(tensors, totals, sizes):
        buf[off:off + size].view(t.shape[0], -1, t.shape[2])[:, :t.shape[1]] = t
        off += size
    return buf


def unpack_planar(out, tensors, totals, world):
    """The gathered [world * per-rank buffer] -> for each tensor of pack_planar its full [L, totals[i], k] (views of out)."""
    out = out.view(world, -1)
    res, off = [], 0
    for t, n in zip(tensors, totals):
        L, per, k = t.shape[0], -(-n // world), t.shape[2]
        res.append(out[:, off:off + L * per * k].reshape(world, L, per, k).transpose(0, 1).reshape(L, world * per, k)[:, :n])
        off += L * per * k
    return res


def all_gather_planar(tensors, total, group=None):
    """Several per-ray tensors of this rank ([count] or [count, k], same count) -> their full versions ([total, ...]) with ONE
    collective (pack_planar)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return list(tensors)
    world = dist.get_world_size(group)
    views = [t.reshape(1, t.shape[0], math.prod(t.shape[1:])) for t in tensors]     # explicit width: empty slices too
    buf = pack_planar(views, [total] * len(views), world)
    out = buf.new_empty(world * buf.numel())                     # concatenated form: accepted by nccl AND gloo
    dist.all_gather_into_tensor(out, buf, group=group)
    full = unpack_planar(out, views, [total] * len(views), world)
    return [f.reshape((total,) + tuple(t.shape[1:])).contiguous() for f, t in zip(full, tensors)]


class _RayPayloadGather(torch.autograd.Function):
    """forward: this rank's [L, count_i, k] slices -> the full [L, totals[i], k] tensors; backward: world x the incoming
    gradient at this rank's own rows (see all_gather_ray_payload)."""

    @staticmethod
    def forward(ctx, spec, *tensors):
        rank, world, totals, collective = spec
        buf = pack_planar(tensors, totals, world, dtype=torch.float64)
        out = buf.new_empty(world * buf.numel())
        collective(out, buf)
        ctx.world = world
        ctx.rows = [ray_slice(n, world, rank) for n in totals]
        ctx.set_materialize_grads(False)
        return tuple(f.to(t.dtype).contiguous() for f, t in zip(unpack_planar(out, tensors, totals, world), tensors))

    @staticmethod
    def backward(ctx, *grads):
        return (None,) + tuple(None if g is None else g[:, b:b + c] * ctx.world for g, (b, c) in zip(grads, ctx.rows))


def all_gather_ray_payload(tensors, totals, rank, world, collective=None, group=None):
    """Per-camera ray payloads of a ray-sharded step -> their full versions on every rank, with ONE collective.

    tensors[i] is this rank's [L, count_i, k] slice of a [L, totals[i], k] tensor: rank r holds rows ray_slice(totals[i],
    world, r) of every one of the L rows (the head's ray_shard gives each rank the same slice of every camera's rays; a
    per-rank scalar is a [1, 1, k] slice of totals[i] = world).  The payload travels in fp64 (exact for fp32 inputs) and comes
    back in each tensor's dtype.  ``collective(out, buf)`` fills ``out`` [world * buf.numel()] with every rank's ``buf`` in
    rank order; default: dist.all_gather_into_tensor over ``group``.

    Gradient contract: every rank evaluates the SAME loss graph on the gathered tensors, so rank r's share of the full
    gradient is the incoming gradient at its own rows.  The backward returns world x that (no collective): parameter
    gradients averaged over the ranks, as DistributedDataParallel does, are then the full gradient."""
    if collective is None:
        def collective(out, buf):
            dist.all_gather_into_tensor(out, buf, group=group)
    return list(_RayPayloadGather.apply((rank, world, list(totals), collective), *tensors))


# ---------------------------------------------------------------------------------------- per-plane row slices of the TPV
# A query-sharded rank owns the contiguous slice ray_slice(Q_i, world, rank) of EACH plane i (sizes = [Q_hw, Q_zh, Q_wz]);
# its rows are those slices one after the other.  For the exchange every slice is padded to ceil(Q_i / world) rows, so all
# ranks send buffers of per_rank_rows(sizes, world) rows.
def plane_slices(sizes, rank, world):
    """[(begin, count)] of this rank in each plane."""
    return [ray_slice(n, world, rank) for n in sizes]


def per_rank_rows(sizes, world):
    return sum(-(-n // world) for n in sizes)


def local_rows(full, sizes, rank, world):
    """This rank's rows out of a [sum(sizes), ...] tensor laid out plane after plane."""
    return local_rows_of(full, sizes, plane_slices(sizes, rank, world))


def local_rows_of(full, sizes, slices):
    """The rows slices [(begin, count)] per plane out of a [sum(sizes), ...] tensor laid out plane after plane."""
    parts, off = [], 0
    for (b, c), n in zip(slices, sizes):
        parts.append(full[off + b:off + b + c])
        off += n
    return torch.cat(parts, 0)


def pad_rows(local, sizes, rank, world):
    """local rows -> [per_rank_rows, C] with each plane's slice padded to ceil(Q_i / world) rows (zeros)."""
    buf = local.new_zeros(per_rank_rows(sizes, world), local.shape[1])
    o_src = o_dst = 0
    for (b, c), n in zip(plane_slices(sizes, rank, world), sizes):
        buf[o_dst:o_dst + c] = local[o_src:o_src + c]
        o_src += c
        o_dst += -(-n // world)
    return buf


def unpad_rows(buf, sizes, rank, world):
    """The inverse of pad_rows: [per_rank_rows, C] -> this rank's rows (padding dropped)."""
    parts, off = [], 0
    for (b, c), n in zip(plane_slices(sizes, rank, world), sizes):
        parts.append(buf[off:off + c])
        off += -(-n // world)
    return torch.cat(parts, 0)


def assemble_rows(gathered, sizes, world):
    """Every rank's padded rows [world, per_rank_rows, C] -> the full planes [sum(sizes), C]."""
    C = gathered.shape[-1]
    out = gathered.new_empty(sum(sizes), C)
    o_dst = o_src = 0
    for n in sizes:
        per = -(-n // world)
        out[o_dst:o_dst + n] = gathered[:, o_src:o_src + per].reshape(world * per, C)[:n]
        o_dst += n
        o_src += per
    return out


def split_rows(full, sizes, world):
    """The inverse of assemble_rows: [sum(sizes), C] -> [world, per_rank_rows, C], rank r's padded rows in block r."""
    C = full.shape[-1]
    out = full.new_zeros(world, per_rank_rows(sizes, world), C)
    o_src = o_dst = 0
    for n in sizes:
        per = -(-n // world)
        plane = full.new_zeros(world * per, C)
        plane[:n] = full[o_src:o_src + n]
        out[:, o_dst:o_dst + per] = plane.view(world, per, C)
        o_src += n
        o_dst += per
    return out


class _RowGather(torch.autograd.Function):
    """forward: this rank's plane rows -> the full planes (one all_gather); backward: this rank's rows of the gradient summed
    over the ranks (one reduce-scatter).  See all_gather_rows."""

    @staticmethod
    def forward(ctx, spec, local):
        sizes, rank, world, collective, reduce_scatter = spec
        buf = pad_rows(local, sizes, rank, world)
        out = buf.new_empty(world * buf.shape[0], buf.shape[1])
        collective(out, buf)
        ctx.spec = spec
        return assemble_rows(out.view(world, buf.shape[0], buf.shape[1]), sizes, world)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        sizes, rank, world, collective, reduce_scatter = ctx.spec
        buf = split_rows(grad.contiguous(), sizes, world)
        out = buf.new_empty(buf.shape[1], buf.shape[2])
        reduce_scatter(out, buf.view(-1, buf.shape[2]))
        return None, unpad_rows(out, sizes, rank, world)


def all_gather_rows(local, sizes, rank, world, collective=None, reduce_scatter=None, group=None):
    """The exchange of the query-sharded encoder, differentiable: this rank's rows [sum(count_i), C] (each plane's slice
    plane_slices(sizes, rank, world), plane after plane) -> the full planes [sum(sizes), C] on every rank.

    Forward: ONE all_gather of the padded slices (pad_rows / assemble_rows).  Backward: ONE reduce-scatter (SUM) of the
    padded incoming gradient (split_rows), whose block for this rank, padding dropped, is the gradient of its rows.
    ``collective(out, buf)`` fills ``out`` [world * rows, C] with every rank's ``buf`` [rows, C] in rank order;
    ``reduce_scatter(out, buf)`` fills ``out`` [rows, C] with the sum over the ranks of block ``rank`` of their ``buf``
    [world * rows, C].  Defaults: dist.all_gather_into_tensor / dist.reduce_scatter_tensor over ``group``.

    Gradient rule: every rank's head and loss give a gradient with respect to the full planes -- partial and already scaled
    by world under head.ray_shard (all_gather_ray_payload), full and unscaled for replicated terms (the sparsity term on
    uniform_sdf).  Either way the sum over the ranks is world x the full gradient, so the reduce-scatter hands rank r
    world x the full gradient at its rows, and the layers below give parameter gradients that are world x rank r's share.
    Everything a rank computes whole (layer 0's input planes, the self-attention value_proj over all rows, the image
    value_projs, the positional-embedding Linear, the image features) receives a partial gradient from that rank's rows,
    and by linearity these too sum to world x the full gradient.  DistributedDataParallel's mean over the ranks is then
    the full gradient, with no extra factor."""
    if collective is None:
        def collective(out, buf):
            dist.all_gather_into_tensor(out, buf, group=group)
    if reduce_scatter is None:
        def reduce_scatter(out, buf):
            dist.reduce_scatter_tensor(out, buf, op=dist.ReduceOp.SUM, group=group)
    sizes = [int(n) for n in sizes]
    n_local = sum(c for _, c in plane_slices(sizes, rank, world))
    if local.dim() != 2 or local.shape[0] != n_local:
        raise ValueError('all_gather_rows: rank %d of %d holds %d rows of planes %s, got %s'
                         % (rank, world, n_local, sizes, tuple(local.shape)))
    return _RowGather.apply((sizes, rank, world, collective, reduce_scatter), local.contiguous())


# ---------------------------------------------------------------------------------------- h-row slabs of the decoded volume
# The decode-sharded training step (head.decode_shard): the volume is H-major (vol_sdf [H, W, zpitch], vol_feat
# [H, W, Z, feat_pitch]), so rank r's slab is rows ray_slice(H, world, r) of both tensors, and the exchange is
# all_gather_rows over ONE plane of H rows whose row is an h row of vol_sdf followed by the same h row of vol_feat.
def volume_slab(H, rank, world):
    """(h_begin, h_count) of this rank's slab of the volume's H rows."""
    if H < world:
        raise ValueError('decode_shard: a volume of %d h rows cannot be split over %d ranks (a rank without rows would leave '
                         'the decode without a gradient there)' % (H, world))
    return ray_slice(H, world, rank)


def pack_volume_rows(vol_sdf, vol_feat):
    """A slab of the volume ([c, W, zpitch], [c, W, Z, feat_pitch] or None) -> the [c, row] rows all_gather_volume sends:
    each row is the slab row of vol_sdf followed by that of vol_feat."""
    c = vol_sdf.shape[0]
    if vol_feat is None:
        return vol_sdf.reshape(c, -1)
    return torch.cat([vol_sdf.reshape(c, -1), vol_feat.reshape(c, -1)], 1)


def volume_exchange_bytes(desc, world):
    """Bytes one decode-sharded step moves per rank through the exchange: the all_gather receives world - 1 padded slabs
    and the reduce-scatter sends as many (ring algorithms; fp32)."""
    row = desc.W * desc.zpitch + (desc.W * desc.Z * desc.feat_pitch if desc.n_feat else 0)
    per = -(-desc.H // world)
    return dict(all_gather=4 * (world - 1) * per * row, reduce_scatter=4 * (world - 1) * per * row)


def all_gather_volume(vol_sdf, vol_feat, H, rank, world, collective=None, reduce_scatter=None, group=None):
    """This rank's slab of the decoded volume (rows volume_slab(H, rank, world) of vol_sdf and vol_feat; vol_feat None when
    no features are decoded) -> the full (vol_sdf, vol_feat) on every rank, contiguous and autograd-connected.

    Forward: ONE all_gather of both tensors' slab rows side by side (pack_volume_rows).  Backward: ONE reduce-scatter (SUM)
    of the full volume gradient, whose block for this rank is the gradient of its slab.  ``collective`` /
    ``reduce_scatter`` / ``group``: as all_gather_rows, over a single plane of H rows.  Gradient rule: as all_gather_rows --
    the sum over the ranks of their volume gradients is world x the full gradient, so this rank's slab receives world x
    its share."""
    b, c = volume_slab(H, rank, world)
    if vol_sdf.shape[0] != c or (vol_feat is not None and vol_feat.shape[0] != c):
        raise ValueError('all_gather_volume: rank %d of %d holds h rows [%d, %d), got a slab of %s'
                         % (rank, world, b, b + c, tuple(vol_sdf.shape)))
    full = all_gather_rows(pack_volume_rows(vol_sdf, vol_feat), [H], rank, world, collective, reduce_scatter, group)
    n_sdf = math.prod(vol_sdf.shape[1:])
    vs = full[:, :n_sdf].reshape(H, *vol_sdf.shape[1:]).contiguous()
    if vol_feat is None:
        return vs, None
    return vs, full[:, n_sdf:].reshape(H, *vol_feat.shape[1:]).contiguous()


def _num_cams(head, metas):
    """Number of cameras the head will render, read from the metas' SHAPES (no copy: usable inside CUDA-graph capture)."""
    import os
    kws = head.img2lidar.trans_kw_eval if os.environ.get('eval', 'false') == 'true' else head.img2lidar.trans_kw
    n = 0
    for k in (kws if isinstance(kws, (list, tuple)) else [kws]):
        v = metas[0][k]
        n += v.shape[0] if hasattr(v, 'shape') else len(v)
    return n


def render_sharded(head, metas, batch=0, group=None):
    """NeuSHead.render with the frame's rays sharded over the process group; every rank returns the
    full maps (bit-identical to the single-GPU render: same kernel, same per-ray arithmetic)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    sampler = head._sampler()
    n_cam = _num_cams(head, metas)
    total = n_cam * sampler.ray_number
    begin, count = ray_slice(total, world, rank)
    out = head.render(metas=metas, batch=batch, ray_range=(begin, count))
    keys = ['ms_depths', 'ms_accs'] + (['ms_max_depths'] if head.return_max_depth else [])
    res = {'ms_rays': out['ms_rays']}
    # one collective: pack the per-ray scalars side by side
    packed = torch.stack([out[k][0] for k in keys], -1)
    full = all_gather_rays(packed, total, group)
    for i, k in enumerate(keys):
        res[k] = [full[:, i].reshape(1, n_cam, sampler.ray_number)]
    return res


def uniform_sdf_sharded(head, aabb, resolution, group=None):
    """Occupancy lattice of NeuSHead.forward_occ / get_uniform_sdf (neus_head.py:265-293) with the lattice points
    sharded over the process group (SURVEY.md 8e, BASELINE configs[3]): each rank queries a contiguous slice of the
    flattened [H, W, D] lattice and ONE all_gather assembles the sdf.  ``head.prepare()`` must have run on every rank."""
    f = head.model.field
    dev = f.vol_sdf.device
    xs = torch.linspace(aabb[0], aabb[3], int((aabb[3] - aabb[0]) / resolution), device=dev)
    ys = torch.linspace(aabb[1], aabb[4], int((aabb[4] - aabb[1]) / resolution), device=dev)
    zs = torch.linspace(aabb[2], aabb[5], int((aabb[5] - aabb[2]) / resolution), device=dev)
    W, H, D = len(xs), len(ys), len(zs)
    xyz = torch.stack([xs[None, :, None].expand(H, W, D), ys[:, None, None].expand(H, W, D),
                       zs[None, None, :].expand(H, W, D)], dim=-1).flatten(0, 2)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = xyz.shape[0]
    begin, count = ray_slice(total, world, rank)
    local = ops.field_query(f.vol_sdf, f.vol_feat, f.desc, xyz[begin:begin + count].contiguous())[0]
    return all_gather_rays(local, total, group).reshape(H, W, D), xyz.reshape(H, W, D, 3)


# ======================================================================================================================
# Strong scaling of ONE frame (SURVEY.md 8e): query-sharded lifting + slab-sharded decode + ray-sharded render.
#
# The reference never shards a frame (DDP replicas only, train.py:86-92).  Inside a frame everything is independent per
# TPV query / voxel / ray EXCEPT that a layer's self-attention reads ALL planes as its value tensor
# (tpvformer_encoder_layer.py:160-183), so the lifting needs one all_gather of the updated planes per layer (30 MB):
#
#   per layer   replicated: value_proj of the image features (3 planes in one GEMM) and of the TPV tokens
#               sharded   : offsets/logits GEMM, self-attention, output_proj(+residual), LayerNorm, per-plane image
#                           cross-attention, output_proj, LayerNorm, FFN, LayerNorm      -- all on this rank's queries
#               exchange  : ONE all_gather of the local token rows
#   decode      each rank decodes a slab of h rows into the full-size volume, ONE all_gather (8.5-33 MB)
#   render      contiguous ray slices (torch.chunk order), ONE all_gather of depth / max-depth / acc / RGB
#
# A rank owns a contiguous 1/world slice of EACH plane (not of the concatenated token sequence): zh / wz queries cost
# ~6x an hw query in the image cross-attention (48 vs 8 pillar points), so slicing per plane balances the visible-pair
# count.  Every kernel is row-independent (a GEMM row, a query, a LayerNorm row depend on nothing else), hence the
# sharded result is BIT-IDENTICAL to the single-GPU encoder -- tests/test_gpu_dist.py checks torch.equal.
class ShardedLifter:
    """Inference-only, bs = 1, post-norm layers ('self_attn','norm','cross_attn','norm','ffn','norm' -- every shipped config)."""

    def __init__(self, encoder):
        from .encoder import POST_NORM_ORDER
        if not hasattr(encoder, 'tpv_size'):
            raise NotImplementedError('ShardedLifter: query-sharded lifting covers the TPV encoder; %s is not sharded'
                                      % type(encoder).__name__)
        self.enc = encoder
        H, W, Z = encoder.tpv_size
        self.sizes = [H * W, Z * H, W * Z]
        for layer in encoder.layers:
            if tuple(layer.operation_order) != POST_NORM_ORDER:
                raise NotImplementedError('ShardedLifter: operation_order %r' % (layer.operation_order,))

    # ---- slices
    def slices(self, rank, world):
        """[(begin, count)] of this rank in each plane."""
        return plane_slices(self.sizes, rank, world)

    def per_rank_rows(self, world):
        return per_rank_rows(self.sizes, world)

    def _local_rows(self, full, rank, world):
        """rows of this rank out of a [Q_total, ...] tensor laid out hw | zh | wz."""
        return local_rows(full, self.sizes, rank, world)

    # ---- per-frame replicated state
    @torch.no_grad()
    def prepare(self, ms_img_feats, metas):
        enc = self.enc
        tpv_pos, feat, shapes, lsi = enc.frame_inputs(ms_img_feats)     # bs = 1, no autograd: the [1, Q_total, C] tensor
        uvs, masks, vises = enc.project_reference_points(metas, feat.device)
        return dict(feat=feat, shapes=shapes, lsi=lsi, uvs=uvs, vises=vises, pos=tpv_pos[0],
                    ref=enc.cross_view_ref_points)                            # [Q_total, 3, P, 2]

    # ---- one layer on this rank's queries
    @torch.no_grad()
    def layer_local(self, li, qfull, st, rank, world):
        """qfull [Q_total, C] (all planes, input of layer li) -> this rank's updated rows [sum(count_i), C]."""
        enc = self.enc
        q = self._local_rows(qfull, rank, world).contiguous()
        if q.shape[0] == 0:
            return q
        return enc.layers[li].forward_rows(q, qfull, self._local_rows(st['pos'], rank, world),
                                           self._local_rows(st['ref'], rank, world), self.slices(rank, world), st['feat'],
                                           st['shapes'], st['lsi'], (enc.tpv_spatial_shapes, enc.tpv_level_start),
                                           st['uvs'], st['vises'])

    # ---- exchange
    def pad_local(self, local, rank, world):
        """local rows -> [per_rank_rows, C] with each plane's slice padded to ceil(Q_i / world) (all_gather needs equal sizes)."""
        return pad_rows(local, self.sizes, rank, world)

    def assemble(self, gathered, world):
        """gathered [world, per_rank_rows, C] -> qfull [Q_total, C]."""
        return assemble_rows(gathered, self.sizes, world)

    @torch.no_grad()
    def forward(self, representation, ms_img_feats, metas, group=None):
        """The encoder's forward on this rank's share; returns the full planes [1, Q_i, C] x 3 on every rank."""
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        st = self.prepare(ms_img_feats, metas)
        qfull = torch.cat([p[0] for p in representation], 0).contiguous()
        for li in range(len(self.enc.layers)):
            local = self.layer_local(li, qfull, st, rank, world)
            if world == 1:
                qfull = local
                continue
            buf = self.pad_local(local, rank, world)
            gathered = buf.new_empty(world * buf.shape[0], buf.shape[1])
            dist.all_gather_into_tensor(gathered, buf, group=group)       # the one exchange of the layer
            qfull = self.assemble(gathered.view(world, buf.shape[0], buf.shape[1]), world)
        return [t[None] for t in torch.split(qfull, self.sizes, 0)]


@torch.no_grad()
def decode_sharded(head, representation, group=None):
    """NeuSHead.prepare with the decode sharded by h rows: every rank decodes ceil(H / world) rows into a volume buffer of
    world * ceil(H / world) rows, ONE all_gather per volume tensor fills in the rest (in place: rank r's rows are the r-th
    block); the field then holds the first H rows as usual."""
    from . import ops as ops_
    f = head.model.field
    if not f.tpv:
        raise NotImplementedError('decode_sharded: the voxel-sharded decode covers the TPV field; tpv=False is not sharded')
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    hw, zh, wz = representation
    l1, l2 = f.density_net[1], f.density_net[3]
    d = f.desc
    if world == 1:
        f.pre_compute_density_color(representation)
        return
    per = -(-d.H // world)
    dev = hw.device
    big_s = torch.empty(world * per, d.W, d.zpitch, device=dev)
    big_f = torch.empty(world * per, d.W, d.Z, d.feat_pitch, device=dev) if d.n_feat else None
    b, c = ray_slice(d.H, world, rank)
    ops_.tpv_decode(hw[0].contiguous(), zh[0].contiguous(), wz[0].contiguous(), l1.weight, l1.bias, l2.weight, l2.bias, d,
                    rows=(b, c), out=(big_s[:d.H], None if big_f is None else big_f[:d.H]))
    dist.all_gather_into_tensor(big_s, big_s[rank * per:(rank + 1) * per].clone(), group=group)
    if big_f is not None:
        dist.all_gather_into_tensor(big_f, big_f[rank * per:(rank + 1) * per].clone(), group=group)
    f.vol_sdf, f.vol_feat = big_s[:d.H], (None if big_f is None else big_f[:d.H])
    f._pack = None


@torch.no_grad()
def frame_sharded(model, ms_img_feats, metas, lifter=None, group=None, batch=0):
    """One frame across the process group: sharded lifting -> sharded decode -> ray-sharded render with ONE final
    all_gather of depth / max-depth / acc (/ RGB).  Returns the full per-ray maps on every rank (flat (cam, ray) order)."""
    lifter = lifter or ShardedLifter(model.encoder)
    rep = model.lifter(ms_img_feats=ms_img_feats)['representation']
    planes = lifter.forward(rep, ms_img_feats, metas, group)
    decode_sharded(model.head, planes, group)
    head = model.head
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n_cam = _num_cams(head, metas)
    total = n_cam * head._sampler().ray_number
    begin, count = ray_slice(total, world, rank)
    out = head.render(metas=metas, batch=batch, ray_range=(begin, count))
    parts, names = [out['ms_depths'][0].reshape(-1), out['ms_accs'][0].reshape(-1)], ['depth', 'acc']
    if head.return_max_depth:
        parts.append(out['ms_max_depths'][0].reshape(-1)); names.append('max_depth')
    if head.model.field.color_dims >= 3:
        parts.append(out['ms_colors'][0].reshape(-1, 3)); names.append('rgb')
    return dict(zip(names, all_gather_planar(parts, total, group)))


class GraphedFrame:
    """frame_sharded captured ONCE into a CUDA graph per rank (kernels + the NCCL all_gathers) and replayed per frame: at high
    rank counts a sharded frame is a few ms of GPU work per rank behind ~110 python-issued launches and 7 collectives, i.e.
    host-bound when run eagerly.  Inputs are static device buffers (copy the frame's FPN features / camera matrices into ``feats`` / ``metas``'
    tensors before ``replay()``); outputs are the static tensors ``self.out``.  ``metas`` must hold DEVICE tensors (a numpy
    matrix list would be uploaded from pageable memory inside the capture).
    STATUS: validated at world size 1 (tests/test_gpu_dist.py, bit-identical to eager).  With torch.distributed's NCCL
    process group inside the capture the first 2-GPU attempt did not complete within the box's time limit (round 2), so
    bench.py uses the graph at N = 1 only and issues eagerly at N > 1 unless ``--graph`` is given."""

    def __init__(self, model, feats, metas, lifter=None, group=None, warmup=2):
        self.model, self.feats, self.metas, self.group = model, feats, metas, group
        self.lifter = lifter or ShardedLifter(model.encoder)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):                       # allocator pools, split-weight caches, NCCL channels
                frame_sharded(model, feats, metas, lifter=self.lifter, group=group)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = frame_sharded(model, feats, metas, lifter=self.lifter, group=group)

    def replay(self):
        self.graph.replay()
        return self.out
