"""Multi-GPU plumbing for the render path (SURVEY.md 8e): rays are independent given the decoded
volume, so the flat (cam, ray) order of neus_head.py:324-325 is split into contiguous per-rank slices
(the same split ``torch.chunk`` produces) and the rendered maps are put back together with ONE
all_gather.  Backend-agnostic (``nccl`` on the GPUs, ``gloo`` in the CPU tests)."""
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


def all_gather_planar(tensors, total, group=None):
    """Several per-ray tensors of this rank ([count] or [count, k], same count) -> their full versions ([total, ...]) with ONE
    collective: the payload is packed PLANAR (tensor after tensor, each padded to the common per-rank length -- contiguous
    copies; an interleaved [count, sum k] pack would cost a strided write of every column)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return list(tensors)
    world = dist.get_world_size(group)
    per = -(-total // world)
    widths = [1 if t.dim() == 1 else t.shape[1] for t in tensors]
    buf = tensors[0].new_zeros(sum(widths) * per)
    off = 0
    for t, w in zip(tensors, widths):
        buf[off:off + t.numel()] = t.reshape(-1)
        off += w * per
    out = buf.new_empty(world * buf.numel())                     # concatenated form: accepted by nccl AND gloo
    dist.all_gather_into_tensor(out, buf, group=group)
    out = out.view(world, buf.numel())
    res, off = [], 0
    for t, w in zip(tensors, widths):
        full = out[:, off:off + w * per].reshape(world * per, *([w] if t.dim() > 1 else []))[:total]
        res.append(full.contiguous())
        off += w * per
    return res


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
        from . import encoder as E
        self.E, self.enc = E, encoder
        H, W, Z = encoder.tpv_size
        self.sizes = [H * W, Z * H, W * Z]
        for layer in encoder.layers:
            if tuple(layer.operation_order) != ('self_attn', 'norm', 'cross_attn', 'norm', 'ffn', 'norm'):
                raise NotImplementedError('ShardedLifter: operation_order %r' % (layer.operation_order,))

    # ---- slices
    def slices(self, rank, world):
        """[(begin, count)] of this rank in each plane."""
        return [ray_slice(n, world, rank) for n in self.sizes]

    def per_rank_rows(self, world):
        return sum(-(-n // world) for n in self.sizes)

    def _local_rows(self, full, rank, world):
        """rows of this rank out of a [Q_total, ...] tensor laid out hw | zh | wz."""
        parts, off = [], 0
        for (b, c), n in zip(self.slices(rank, world), self.sizes):
            parts.append(full[off + b:off + b + c])
            off += n
        return torch.cat(parts, 0)

    # ---- per-frame replicated state
    @torch.no_grad()
    def prepare(self, ms_img_feats, metas):
        enc = self.enc
        feat, shapes, lsi = enc.flatten_features(ms_img_feats)
        dev = feat.device
        uvs, masks, vises = enc.project_reference_points(metas, dev)
        pv = enc._tpv_pos()
        pos = enc._pos_cat[0] if getattr(enc, '_pos_val', None) is pv else torch.cat(list(pv), 0)      # [Q_total, C]
        return dict(feat=feat, shapes=shapes, lsi=lsi, uvs=uvs, vises=vises, pos=pos,
                    ref=enc.cross_view_ref_points)                            # [Q_total, 3, P, 2]

    # ---- one layer on this rank's queries
    @torch.no_grad()
    def layer_local(self, li, qfull, st, rank, world):
        """qfull [Q_total, C] (all planes, input of layer li) -> this rank's updated rows [sum(count_i), C]."""
        E, ops_ = self.E, ops
        layer = self.enc.layers[li]
        sa, ca = layer.attentions[0], layer.attentions[1]
        sl = self.slices(rank, world)
        q = self._local_rows(qfull, rank, world).contiguous()
        if q.shape[0] == 0:
            return q
        Hd, L, P = sa.num_heads, sa.num_levels, sa.num_points
        # -- self attention (cross_view_hybrid_attention.py:63-124): value = ALL tokens, queries = local rows (+ pos)
        v = E.fast_linear(sa.value_proj, qfull)
        qp = q + self._local_rows(st['pos'], rank, world)
        _, (offs, logits) = E.fast_linear_cat(sa, '_so_offlog', [sa.sampling_offsets, sa.attention_weights], qp)
        ref = self._local_rows(st['ref'], rank, world).contiguous()
        out = ops_.tpv_self_attn_forward_rows(v, Hd, v.shape[1] // Hd, self.enc.tpv_spatial_shapes, self.enc.tpv_level_start,
                                              offs, logits, ref, L, P)
        q = E.fast_linear(sa.output_proj, out, residual=q, ln=layer.norms[0])
        # -- image cross attention, one plane at a time (tpvformer/attention/image_cross_attention.py:83-93)
        feat = st['feat']
        n_cam, nv = feat.shape[0], feat.shape[1]
        vps = [a.deformable_attention.value_proj for a in ca.attns]
        _, vrows = E.fast_linear_cat(ca, '_so_value3', vps, feat[:, :, 0].reshape(-1, feat.shape[-1]))
        outs, o0 = [], 0
        for i, (b, c) in enumerate(sl):
            if c == 0:
                continue
            att = ca.attns[i]
            da = att.deformable_attention
            qi = q[o0:o0 + c]
            _, (offs, logits) = E.fast_linear_cat(da, '_so_offlog', [da.sampling_offsets, da.attention_weights], qi)
            uv = st['uvs'][i][:, 0, b:b + c].contiguous()
            vis = st['vises'][i][:, b:b + c].contiguous()
            slots = ops_.tpv_cross_attn_forward_rows(vrows[i], n_cam, da.num_heads, qi.shape[1] // da.num_heads, st['shapes'], st['lsi'],
                                                     offs, logits, uv, vis, da.num_levels, da.num_points)
            outs.append(E.fast_linear(att.output_proj, slots, residual=qi, ln=layer.norms[1]))
            o0 += c
        q = torch.cat(outs, 0)
        ffn = layer.ffns[0]
        h = E.fast_linear(ffn.layers[0][0], q, relu=True)
        return E.fast_linear(ffn.layers[1], h, residual=q if ffn.add_identity else None, ln=layer.norms[2])

    # ---- exchange
    def pad_local(self, local, rank, world):
        """local rows -> [per_rank_rows, C] with each plane's slice padded to ceil(Q_i / world) (all_gather needs equal sizes)."""
        C = local.shape[1]
        buf = local.new_zeros(self.per_rank_rows(world), C)
        o_src = o_dst = 0
        for (b, c), n in zip(self.slices(rank, world), self.sizes):
            buf[o_dst:o_dst + c] = local[o_src:o_src + c]
            o_src += c
            o_dst += -(-n // world)
        return buf

    def assemble(self, gathered, world):
        """gathered [world, per_rank_rows, C] -> qfull [Q_total, C]."""
        C = gathered.shape[-1]
        out = gathered.new_empty(sum(self.sizes), C)
        o_dst = o_src = 0
        for n in self.sizes:
            per = -(-n // world)
            out[o_dst:o_dst + n] = gathered[:, o_src:o_src + per].reshape(world * per, C)[:n]
            o_dst += n
            o_src += per
        return out

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
