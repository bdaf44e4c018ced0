"""A2-A11: TPVFormer encoder behind the reference's module API.

Class names, constructor kwargs, forward signatures, output dict keys and ``state_dict`` key names
follow the reference (file:line in each docstring) so that configs and checkpoints carry over.
The arithmetic of the hot ops runs in ``libselfocc_b200.so``:

* inference (eval, no autograd, batch 1, post-norm layers -- every shipped config): ``TPVFormerLayer.forward_rows``,
  one routine per layer shared with the query-sharded lifter (``dist.ShardedLifter``).  One fused kernel per attention --
  softmax + sampling-location arithmetic + bilinear gather + head sum (+ camera loop / visible-count average for the
  image cross-attention), no ``nonzero()`` host sync, no padded per-camera rebatch (``ops.tpv_self_attn_forward_rows`` /
  ``ops.tpv_cross_attn_forward_rows``); every dense projection (value / offset / weight / output Linear, FFN) runs on
  the wgmma split-precision GEMM (``ops.linear_3xtf32``, fp32-level accuracy), projections of the same input are
  fused into one GEMM, and each LayerNorm is folded into the epilogue of the GEMM before it;
* training (autograd, or train mode), batch 1, post-norm layers: ``TPVFormerLayer.forward_rows_train``, one routine per
  layer on all rows, or on the rank's rows of each plane in the query-sharded step (``TPVFormerEncoder.query_shard =
  (rank, world)``, one ``dist.all_gather_rows`` per layer).  The same fused attention cores with their backward kernels
  (``ops.TPVSelfAttnFunction`` / ``ops.TPVCrossAttnFunction``: no host sync, no padded rebatch, no sampling-location
  tensor); the projections run forward and input gradient on the wgmma GEMM (``train_linear``), the weight gradients on
  cuBLAS;
* batch > 1 or a ``key_padding_mask``: the attention modules' own forwards, the reference's formulation: the mmcv-contract op
  ``ops.MultiScaleDeformableAttnFunction`` fed by torch softmax / location arithmetic, with the image
  cross-attention's rebatch built from device-compacted index lists (``ops.visible_index_lists``).
"""
import copy
import math
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .mapping import GridMeterMapping
from .registry import MODELS, HAVE_MMENGINE, build_attention, build_positional_encoding, build_transformer_layer


# --------------------------------------------------------------------------- construction-time tables
def _pillar_tables(mapping, num_points_cross):
    """Per-plane pillars of 3-D reference points in metres, [P, Q, 3] each
    (tpvformer_encoder.py:131-154; ``num_points_cross`` = [p_wz, p_zh, p_hw])."""
    H, W, Z = mapping.size_h, mapping.size_w, mapping.size_d
    p_hw, p_zh, p_wz = num_points_cross[2], num_points_cross[1], num_points_cross[0]
    f = lambda n: torch.arange(n, dtype=torch.float)

    def table(dims, p, h_idx, w_idx, d_idx):
        g = torch.empty(*dims, p, 3)
        g[..., 0], g[..., 1], g[..., 2] = h_idx, w_idx, d_idx
        return mapping.grid2meter(g).reshape(-1, p, 3).transpose(0, 1).contiguous()

    hw = table((H, W), p_hw, f(H)[:, None, None], f(W)[None, :, None], torch.linspace(0, Z - 1, p_hw)[None, None, :])
    zh = table((Z, H), p_zh, f(H)[None, :, None], torch.linspace(0, W - 1, p_zh)[None, None, :], f(Z)[:, None, None])
    wz = table((W, Z), p_wz, torch.linspace(0, H - 1, p_wz)[None, None, :], f(W)[:, None, None], f(Z)[None, :, None])
    return hw, zh, wz


def _cross_view_refs(H, W, Z, P):
    """[HW+ZH+WZ, 3, P, 2] normalised (x, y) reference points of every query on each of the three
    planes (tpvformer/utils.py:5-71): in-plane coordinates are cell/size, the missing axis is a pillar
    of P points ``linspace(0, size-1, P)/size``."""
    cell = {'h': torch.arange(H, dtype=torch.float) / H, 'w': torch.arange(W, dtype=torch.float) / W,
            'z': torch.arange(Z, dtype=torch.float) / Z}
    size = {'h': H, 'w': W, 'z': Z}
    # level (plane) -> (x axis, y axis):  hw -> (w, h), zh -> (h, z), wz -> (z, w)
    level_axes = (('w', 'h'), ('h', 'z'), ('z', 'w'))
    out = []
    for q_axes in (('h', 'w'), ('z', 'h'), ('w', 'z')):       # query plane, row-major over (first, second)
        n0, n1 = size[q_axes[0]], size[q_axes[1]]
        missing = ({'h', 'w', 'z'} - set(q_axes)).pop()
        coord = {q_axes[0]: cell[q_axes[0]][:, None, None].expand(n0, n1, P),
                 q_axes[1]: cell[q_axes[1]][None, :, None].expand(n0, n1, P),
                 missing: (torch.linspace(0, size[missing] - 1, P) / size[missing])[None, None, :].expand(n0, n1, P)}
        lv = [torch.stack([coord[ax], coord[ay]], -1) for ax, ay in level_axes]
        out.append(torch.stack(lv, 2).reshape(n0 * n1, 3, P, 2))
    return torch.cat(out, 0)


def _metas_matrix(metas, key, device):
    """metas[b][key] (list of N 4x4 arrays / tensors, as the dataset emits them) -> [B, N, 4, 4] fp32 on
    ``device`` (bevformer/utils.py:119-126, img2lidar.py:36-47)."""
    mats = []
    for m in metas:
        v = m[key]
        if isinstance(v, torch.Tensor):
            mats.append(v.to(device=device, dtype=torch.float32))
        elif isinstance(v[0], torch.Tensor):
            mats.append(torch.stack([t.to(device=device, dtype=torch.float32) for t in v]))
        else:
            mats.append(torch.as_tensor(np.asarray(v), dtype=torch.float32, device=device))
    return torch.stack(mats)


_FOCAL_KEYS = ('focal_ratios_x', 'focal_ratios_y')


def _focal_scale(metas, n_cam, device):
    """metas[0]['focal_ratios_x' / '_y'] -> scale_xy [n_cam, 2] fp32 on ``device``, or None when the metas carry neither.

    RandomScaleImageMultiViewImage (dataset/transform_3d.py:362-363) writes both as lists of Python floats; numpy arrays and
    tensors are taken too.  Like the reference (bevformer/utils.py:198-204) only metas[0]'s ratios are read, rounded to fp32
    as ``new_tensor`` does, and a length of 1 broadcasts over the cameras.  A tensor already on ``device`` is used without
    a host copy, so a captured graph (dist.GraphedFrame) reads whatever ratios were written into it before a replay.
    Raises ValueError, before any kernel launch, for one key without the other or a length other than 1 or n_cam."""
    m = metas[0]
    present = [k in m for k in _FOCAL_KEYS]
    if not any(present):
        return None
    if not all(present):
        raise ValueError('metas[0] has %s without %s: the focal-ratio rescale needs both'
                         % (_FOCAL_KEYS[present.index(True)], _FOCAL_KEYS[present.index(False)]))
    cols = []
    for k in _FOCAL_KEYS:
        v = m[k]
        if isinstance(v, torch.Tensor):
            t = v.reshape(-1)
        else:
            t = torch.as_tensor(np.asarray(v, dtype=np.float64).reshape(-1))
        if t.numel() not in (1, n_cam):
            raise ValueError('metas[0][%r] holds %d ratios for %d cameras (expected 1 or %d)' % (k, t.numel(), n_cam, n_cam))
        cols.append(t.to(device=device, dtype=torch.float32).expand(n_cam))
    return torch.stack(cols, -1)


# --------------------------------------------------------------------------- positional encoding (A10)
@MODELS.register_module()
class TPVPositionalEncoding(nn.Module):
    """tpvformer_pos_embed.py:16-58: sin/cos of range-normalised plane metres -> Linear per plane."""

    def __init__(self, num_freqs, embed_dims, tpv_meters, tot_range, init_cfg=None):
        super().__init__()
        assert isinstance(tot_range, (list, tuple)) and len(tot_range) == 6
        r = [float(v) for v in tot_range]
        norm = {'x': (r[0], r[3] - r[0]), 'y': (r[1], r[4] - r[1]), 'z': (r[2], r[5] - r[2])}
        for name, meter, axes, nf in zip(('hw', 'zh', 'wz'), tpv_meters, ('xy', 'yz', 'xz'), num_freqs):
            m = torch.stack([(meter[..., i] - norm[a][0]) / norm[a][1] for i, a in enumerate(axes)], -1)
            freqs = math.pi * (2.0 ** torch.arange(-1, nf - 1, dtype=torch.float))
            ang = m.unsqueeze(-1) * freqs                                  # [A, B, 2, nf]
            feat = torch.stack([ang.sin(), ang.cos()], -1).flatten(-3).flatten(0, 1)
            self.register_buffer(name + '_freq_feat', feat, False)
            setattr(self, 'position_layer_' + name, nn.Linear(4 * nf, embed_dims))

    def forward(self):
        return [self.position_layer_hw(self.hw_freq_feat), self.position_layer_zh(self.zh_freq_feat),
                self.position_layer_wz(self.wz_freq_feat)]


# --------------------------------------------------------------------------- attention modules
def _ring_bias(num_heads, num_levels, num_points, scale_points):
    """sampling_offsets bias init: unit ring over heads (image_cross_attention.py:228-241); mmcv's
    MultiScaleDeformableAttention additionally scales point i by (i + 1)."""
    th = torch.arange(num_heads, dtype=torch.float32) * (2.0 * math.pi / num_heads)
    g = torch.stack([th.cos(), th.sin()], -1)
    g = (g / g.abs().max(-1, keepdim=True)[0]).view(num_heads, 1, 1, 2).repeat(1, num_levels, num_points, 1)
    if scale_points:
        g = g * torch.arange(1, num_points + 1, dtype=torch.float32).view(1, 1, -1, 1)
    return g.reshape(-1)


class _DeformBase(nn.Module):
    def __init__(self, embed_dims, num_heads, num_levels, num_points, im2col_step, value_proj_ratio=1.0):
        super().__init__()
        if embed_dims % num_heads != 0:
            raise ValueError('embed_dims must be divisible by num_heads, but got %d and %d' % (embed_dims, num_heads))
        self.embed_dims, self.num_heads, self.num_levels, self.num_points = embed_dims, num_heads, num_levels, num_points
        self.im2col_step = im2col_step
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, int(embed_dims * value_proj_ratio))

    def _init_common(self, scale_points):
        nn.init.constant_(self.sampling_offsets.weight, 0.)
        with torch.no_grad():
            self.sampling_offsets.bias.copy_(_ring_bias(self.num_heads, self.num_levels, self.num_points, scale_points))
        nn.init.constant_(self.attention_weights.weight, 0.)
        nn.init.constant_(self.attention_weights.bias, 0.)
        nn.init.xavier_uniform_(self.value_proj.weight)
        nn.init.constant_(self.value_proj.bias, 0.)


def fast_linear(lin, x, relu=False, residual=None, out=None, ln=None):
    """nn.Linear forward for the inference path: the wgmma split-precision GEMM (``so_linear_3xtf32``) when the shape
    allows it (K % 96 == 0), cuBLAS otherwise.  Split weights are cached per parameter version.
    ``ln``: an nn.LayerNorm applied to the result; folded into the GEMM epilogue when the row fits one tile
    (``so_linear_3xtf32_ln``), a separate ``so_layer_norm`` launch otherwise."""
    if ln is not None:
        N, K = lin.weight.shape
        if x.is_cuda and x.dtype == torch.float32 and ops.linear_ln_supported(N, K):
            return _fast_linear_impl(lin, x, relu, residual, out, (ln.weight.detach(), ln.bias.detach(), ln.eps))
        y = _fast_linear_impl(lin, x, relu, residual, None, None)
        if y.is_cuda and y.dtype == torch.float32 and y.shape[-1] <= 256:
            y = ops.layer_norm(y.contiguous(), ln.weight.detach(), ln.bias.detach(), ln.eps)
        else:
            y = ln(y)
        if out is not None:
            out.copy_(y.view_as(out))
            return out
        return y
    return _fast_linear_impl(lin, x, relu, residual, out, None)


def _fast_linear_impl(lin, x, relu, residual, out, ln):
    w = lin.weight
    if x.is_cuda and x.dtype == torch.float32 and ops.linear_supported(w.shape[1], w.shape[0]):
        ver = (w._version, w.data_ptr())
        ent = getattr(lin, '_so_split', None)       # kept on the module itself: no aliasing between models
        if ent is None or ent[0] != ver:
            with torch.no_grad():
                ent = (ver,) + ops.split_tf32(w.detach().contiguous())
            lin._so_split = ent
        return ops.linear_3xtf32(x.contiguous(), ent[1], ent[2], lin.bias.detach() if lin.bias is not None else None,
                                 relu=relu, residual=None if residual is None else residual.contiguous(), out=out, ln=ln)
    assert ln is None
    y = F.linear(x, w, lin.bias)
    if relu:
        y = F.relu(y)
    y = y if residual is None else y + residual
    if out is not None:
        out.copy_(y.view_as(out))
        return out
    return y


def train_linear(lin, x):
    """nn.Linear inside the autograd (training) path: forward and input gradient on the wgmma 3xTF32 GEMM
    (ops.TCLinearFunction) when the shape allows it, the stock nn.Linear otherwise."""
    w = lin.weight
    if x.is_cuda and x.dtype == torch.float32 and w.dtype == torch.float32 and x.numel() > 0 \
            and ops.linear_supported(w.shape[1], w.shape[0]) and _needs_grad(x, w):
        return ops.TCLinearFunction.apply(x, w, lin.bias)
    return lin(x)


def fast_linear_cat(owner, key, lins, x):
    """Several nn.Linear layers applied to the SAME input as one wgmma GEMM (weights concatenated along N, cached on
    ``owner``).  Returns the [M, sum(N_i)] result and the column slices (views, unit column stride) of each layer."""
    ver = tuple((l.weight._version, l.weight.data_ptr(), l.bias._version, l.bias.data_ptr()) for l in lins)
    ent = getattr(owner, key, None)
    if ent is None or ent[0] != ver:
        with torch.no_grad():
            w = torch.cat([l.weight.detach() for l in lins], 0).contiguous()
            b = torch.cat([l.bias.detach() for l in lins], 0).contiguous()
            hi, lo = ops.split_tf32(w)
        ent = (ver, hi, lo, b, [l.weight.shape[0] for l in lins])
        setattr(owner, key, ent)
    y = ops.linear_3xtf32(x.contiguous(), ent[1], ent[2], ent[3])
    outs, c0 = [], 0
    for n in ent[4]:
        outs.append(y[:, c0:c0 + n])
        c0 += n
    return y, outs


def _fusable(lins, x):
    return x.is_cuda and x.dtype == torch.float32 and all(ops.linear_supported(l.weight.shape[1], l.weight.shape[0]) for l in lins)


def _offsets_logits(da, x):
    """sampling_offsets(x), attention_weights(x) of a deformable attention as [n, *] row views: one GEMM when both shapes
    allow it, two otherwise."""
    lins = [da.sampling_offsets, da.attention_weights]
    if _fusable(lins, x):
        return fast_linear_cat(da, '_so_offlog', lins, x)[1]
    return fast_linear(lins[0], x), fast_linear(lins[1], x)


def _needs_grad(*tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _cuda_fp32(*tensors):
    return all(t.is_cuda and t.dtype == torch.float32 for t in tensors)


@MODELS.register_module()
class CrossViewHybridAttention(_DeformBase):
    """A8.  cross_view_hybrid_attention.py:11-124 (subclass of mmcv MultiScaleDeformableAttention whose
    only change is the per-point reference broadcast, :96-99).  Parameters: sampling_offsets,
    attention_weights, value_proj, output_proj.  forward is the reference's formulation, for the layers that do not run a
    row routine (batch > 1, a key_padding_mask); TPVFormerLayer runs this attention's batch-1 arithmetic itself."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64, dropout=0.1,
                 batch_first=False, norm_cfg=None, init_cfg=None, value_proj_ratio=1.0, **kwargs):
        super().__init__(embed_dims, num_heads, num_levels, num_points, im2col_step, value_proj_ratio)
        self.batch_first = batch_first
        self.dropout = nn.Dropout(dropout)
        self.output_proj = nn.Linear(int(embed_dims * value_proj_ratio), embed_dims)
        self.init_weights()

    def init_weights(self):
        self._init_common(scale_points=True)
        nn.init.xavier_uniform_(self.output_proj.weight)
        nn.init.constant_(self.output_proj.bias, 0.)

    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, level_start_index=None, **kwargs):
        if value is None:
            value = query
        if identity is None:
            identity = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, num_query, _ = query.shape
        num_value = value.shape[1]
        Hd, L, P = self.num_heads, self.num_levels, self.num_points
        if reference_points.shape[-1] != 2:
            raise ValueError('Last dim of reference_points must be 2, but get %d instead.' % reference_points.shape[-1])
        value = train_linear(self.value_proj, value)
        if key_padding_mask is not None:
            value = value.masked_fill(key_padding_mask[..., None], 0.0)
        value = value.view(bs, num_value, Hd, -1)
        offsets = train_linear(self.sampling_offsets, query).view(bs, num_query, Hd, L, P, 2)
        logits = train_linear(self.attention_weights, query).view(bs, num_query, Hd, L * P)
        aw = logits.softmax(-1).view(bs, num_query, Hd, L, P)
        normalizer = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1).to(offsets.dtype)
        loc = reference_points[:, :, None, :, :, :] + offsets / normalizer[None, None, None, :, None, :]
        out = ops.MultiScaleDeformableAttnFunction.apply(value, spatial_shapes, level_start_index, loc, aw, self.im2col_step)
        out = train_linear(self.output_proj, out)
        if not self.batch_first:
            out = out.permute(1, 0, 2)
        return self.dropout(out) + identity


@MODELS.register_module()
class BEVDeformableAttention(_DeformBase):
    """A6/A7.  image_cross_attention.py:148-351: value_proj / sampling_offsets / attention_weights,
    one offset per pillar point (num_points == D); no output_proj, no residual."""

    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64, dropout=0.1,
                 batch_first=False, norm_cfg=None, init_cfg=None, value_proj_ratio=1.0, **kwargs):
        super().__init__(embed_dims, num_heads, num_levels, num_points, im2col_step, value_proj_ratio)
        self.batch_first = batch_first
        self.init_weights()

    def init_weights(self):
        self._init_common(scale_points=False)

    def forward(self, query, key=None, value=None, identity=None, query_pos=None, key_padding_mask=None,
                reference_points=None, spatial_shapes=None, level_start_index=None, **kwargs):
        """The reference's padded-rebatch contract: query [B*N, Lmax, C], reference_points [B*N, Lmax, D, 2]."""
        if value is None:
            value = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        bs, num_query, _ = query.shape
        num_value = value.shape[1]
        Hd, L, P = self.num_heads, self.num_levels, self.num_points
        value = train_linear(self.value_proj, value)
        if key_padding_mask is not None:
            value = value.masked_fill(key_padding_mask[..., None], 0.0)
        value = value.view(bs, num_value, Hd, -1)
        offsets = train_linear(self.sampling_offsets, query).view(bs, num_query, Hd, L, P, 2)
        aw = train_linear(self.attention_weights, query).view(bs, num_query, Hd, L * P).softmax(-1).view(bs, num_query, Hd, L, P)
        if reference_points.shape[-1] != 2:
            raise ValueError('Last dim of reference_points must be 2, but get %d instead.' % reference_points.shape[-1])
        normalizer = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1).to(offsets.dtype)
        loc = reference_points[:, :, None, None, :, :] + offsets / normalizer[None, None, None, :, None, :]
        out = ops.MultiScaleDeformableAttnFunction.apply(value.contiguous(), spatial_shapes, level_start_index,
                                                         loc.contiguous(), aw.contiguous(), self.im2col_step)
        if not self.batch_first:
            out = out.permute(1, 0, 2)
        return out


@MODELS.register_module()
class BEVCrossAttention(nn.Module):
    """A5.  image_cross_attention.py:11-139.  forward reproduces the reference's rebatch with device-compacted index
    lists, for the layers that do not run a row routine (batch > 1, a key_padding_mask); TPVFormerLayer runs this
    attention's batch-1 arithmetic itself, on the rebatch-free fused core."""

    def __init__(self, embed_dims=256, num_cams=6, dropout=0.1, init_cfg=None, batch_first=True,
                 deformable_attention=dict(type='BEVDeformableAttention', embed_dims=256, num_levels=4), **kwargs):
        super().__init__()
        self.dropout = nn.Dropout(dropout)
        self.deformable_attention = build_attention(deformable_attention)
        self.embed_dims, self.num_cams, self.batch_first = embed_dims, num_cams, batch_first
        self.output_proj = nn.Linear(embed_dims, embed_dims)
        self.init_weight()

    def init_weight(self):
        nn.init.xavier_uniform_(self.output_proj.weight)
        nn.init.constant_(self.output_proj.bias, 0.)

    def forward(self, query, key, value, residual=None, spatial_shapes=None, reference_points_cams=None,
                bev_masks=None, level_start_index=None, **kwargs):
        """query [B,Q,C]; key/value [N, sum(hw), B, C]; reference_points_cams [N,B,Q,D,2];
        bev_masks [N,B,Q,D] (bool/uint8)."""
        if key is None:
            key = query
        if value is None:
            value = key
        if residual is None:
            residual = query
        assert reference_points_cams.size(3) == self.deformable_attention.num_points
        slots = self._rebatch_forward(query, value, spatial_shapes, reference_points_cams, bev_masks, level_start_index)
        slots = train_linear(self.output_proj, slots)
        return self.dropout(slots) + residual

    def _rebatch_forward(self, query, value, spatial_shapes, ref_cams, masks, level_start_index):
        bs, num_query, C = query.shape
        D = ref_cams.size(3)
        lists, lens = ops.visible_index_lists(masks[:, 0].to(torch.uint8).contiguous())   # device-side nonzero()
        lens = lens.tolist()                                                            # one sync (sizes the rebatch)
        max_len = max(lens)
        q_re = query.new_zeros(bs * self.num_cams, max_len, C)
        r_re = ref_cams.new_zeros(bs * self.num_cams, max_len, D, 2)
        idx = [lists[i, :lens[i]] for i in range(self.num_cams)]
        for i in range(self.num_cams):
            for j in range(bs):
                q_re[j * self.num_cams + i, :lens[i]] = query[j, idx[i]]
                r_re[j * self.num_cams + i, :lens[i]] = ref_cams[i, j, idx[i]]
        n_cam, l, _, _ = value.shape
        v = value.permute(2, 0, 1, 3).reshape(self.num_cams * bs, l, C)
        out = self.deformable_attention(query=q_re, key=v, value=v, reference_points=r_re, spatial_shapes=spatial_shapes,
                                        level_start_index=level_start_index)
        slots = torch.zeros_like(query)
        for i in range(self.num_cams):
            for j in range(bs):
                slots[j] = slots[j].index_add(0, idx[i], out[j * self.num_cams + i, :lens[i]])
        count = (masks.sum(-1) > 0).permute(1, 2, 0).sum(-1).clamp(min=1.0)
        return slots / count[..., None]


@MODELS.register_module()
class TPVCrossAttention(nn.Module):
    """tpvformer/attention/image_cross_attention.py:6-96: one BEVCrossAttention per plane with
    num_points = num_points[2], [1], [0] for hw, zh, wz."""

    def __init__(self, embed_dims=256, num_cams=6, dropout=0.1, init_cfg=None, batch_first=True, num_heads=16,
                 num_levels=4, num_points=[64, 64, 8], **kwargs):
        super().__init__()
        self.embed_dims = embed_dims

        def plane(p):
            return build_attention(dict(
                type='BEVCrossAttention', embed_dims=embed_dims, num_cams=num_cams, dropout=dropout, batch_first=batch_first,
                deformable_attention=dict(type='BEVDeformableAttention', embed_dims=embed_dims, num_heads=num_heads,
                                          num_levels=num_levels, num_points=p, dropout=dropout, batch_first=batch_first)))
        self.attn_hw, self.attn_zh, self.attn_wz = plane(num_points[2]), plane(num_points[1]), plane(num_points[0])
        self.attns = [self.attn_hw, self.attn_zh, self.attn_wz]

    def forward(self, query, key, value, residual=None, spatial_shapes=None, reference_points_cams=None, tpv_masks=None,
                level_start_index=None, **kwargs):
        return [self.attns[i](query[i], key, value, residual[i] if residual is not None else None,
                              spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                              reference_points_cams=reference_points_cams[i], bev_masks=tpv_masks[i])
                for i in range(3)]


class FFN(nn.Module):
    """mmcv.cnn.bricks.transformer.FFN with num_fcs=2 (same parameter names: layers.0.0, layers.1)."""

    def __init__(self, embed_dims=256, feedforward_channels=1024, num_fcs=2, act_cfg=dict(type='ReLU', inplace=True),
                 ffn_drop=0., dropout_layer=None, add_identity=True, init_cfg=None, **kwargs):
        super().__init__()
        assert num_fcs == 2, 'only the 2-layer FFN used by the SelfOcc configs is implemented'
        if act_cfg.get('type', 'ReLU') != 'ReLU':
            raise NotImplementedError('FFN activation %r' % (act_cfg,))
        self.embed_dims, self.feedforward_channels, self.add_identity = embed_dims, feedforward_channels, add_identity
        self.layers = nn.Sequential(
            nn.Sequential(nn.Linear(embed_dims, feedforward_channels), nn.ReLU(inplace=True), nn.Dropout(ffn_drop)),
            nn.Linear(feedforward_channels, embed_dims), nn.Dropout(ffn_drop))

    def forward(self, x, identity=None):
        l0 = self.layers[0]
        out = self.layers[2](train_linear(self.layers[1], l0[2](F.relu(train_linear(l0[0], x)))))
        if not self.add_identity:
            return out
        return (x if identity is None else identity) + out


if not HAVE_MMENGINE:  # mmcv registers its own FFN when present
    MODELS.register_module(name='FFN', module=FFN)


POST_NORM_ORDER = ('self_attn', 'norm', 'cross_attn', 'norm', 'ffn', 'norm')     # every shipped config's layer


def _whole(views, split):
    """The concatenated [B, sum(split), C] tensor when `views` are exactly its torch.split pieces, else None."""
    base = getattr(views[0], '_base', None)
    if base is None or base.dim() != 3 or base.shape[1] != sum(split) or not base.is_contiguous():
        return None
    if base.shape[0] != 1 or len(views) != len(split):
        return None
    off = 0
    for v, n in zip(views, split):
        if v._base is not base or v.shape != (1, n, base.shape[2]) or v.stride() != base.stride() \
                or v.data_ptr() != base.data_ptr() + off * base.shape[2] * base.element_size():
            return None
        off += n
    return base


@MODELS.register_module()
class TPVFormerLayer(nn.Module):
    """A9.  tpvformer_encoder_layer.py:9-219."""

    def __init__(self, attn_cfgs=None, ffn_cfgs=dict(type='FFN', feedforward_channels=1024, num_fcs=2, ffn_drop=0.,
                                                     act_cfg=dict(type='ReLU', inplace=True)),
                 operation_order=None, norm_cfg=dict(type='LN'), init_cfg=None, batch_first=True,
                 multi_plane_ffn_norm=False, **kwargs):
        super().__init__()
        ffn_cfgs = copy.deepcopy(ffn_cfgs)
        for old, new in dict(feedforward_channels='feedforward_channels', ffn_dropout='ffn_drop', ffn_num_fcs='num_fcs').items():
            if old in kwargs:
                ffn_cfgs[new] = kwargs[old]
        if multi_plane_ffn_norm:
            raise NotImplementedError('multi_plane_ffn_norm=True is disabled in every shipped config')
        if norm_cfg.get('type', 'LN') != 'LN':
            raise NotImplementedError('norm_cfg %r' % (norm_cfg,))
        self.batch_first, self.multi_plane_ffn_norm = batch_first, multi_plane_ffn_norm
        num_attn = operation_order.count('self_attn') + operation_order.count('cross_attn')
        if isinstance(attn_cfgs, dict):
            attn_cfgs = [copy.deepcopy(attn_cfgs) for _ in range(num_attn)]
        assert num_attn == len(attn_cfgs)
        self.num_attn, self.operation_order, self.norm_cfg = num_attn, operation_order, norm_cfg
        self.pre_norm = operation_order[0] == 'norm'
        self.attentions = nn.ModuleList()
        for name, cfg in zip([o for o in operation_order if o in ('self_attn', 'cross_attn')], attn_cfgs):
            cfg = copy.deepcopy(cfg)
            assert cfg.setdefault('batch_first', batch_first) == batch_first
            att = build_attention(cfg)
            att.operation_name = name
            self.attentions.append(att)
        self.embed_dims = self.attentions[0].embed_dims
        num_ffns = operation_order.count('ffn')
        if isinstance(ffn_cfgs, dict):
            ffn_cfgs = [copy.deepcopy(ffn_cfgs) for _ in range(num_ffns)]
        self.ffns = nn.ModuleList()
        for c in ffn_cfgs:
            c = {k: v for k, v in c.items() if k != 'type'}
            assert c.setdefault('embed_dims', self.embed_dims) == self.embed_dims
            self.ffns.append(FFN(**c))
        self.norms = nn.ModuleList([nn.LayerNorm(self.embed_dims) for _ in range(operation_order.count('norm'))])

    def forward(self, query, key=None, value=None, tpv_pos=None, ref_2d=None, spatial_shapes=None, level_start_index=None,
                reference_points_cams=None, tpv_masks=None, tpv_size=None, tpv_vis=None, tpv_levels=None, **kwargs):
        H, W, Z = tpv_size
        split = [H * W, Z * H, W * Z]
        dev = query[0].device
        if tpv_levels is None:   # tpvformer_encoder_layer.py:160-166
            ss = torch.tensor([[H, W], [Z, H], [W, Z]], device=dev)
            tpv_levels = (ss, torch.tensor([0, H * W, H * W + Z * H], device=dev))
        pos_cat = torch.cat(tpv_pos, dim=1) if isinstance(tpv_pos, (list, tuple)) else tpv_pos
        routine = self._row_routine(query[0], value, kwargs)
        if routine is not None:
            if tpv_vis is None:
                tpv_vis = [(m[:, 0].sum(-1) > 0).to(torch.uint8) for m in tpv_masks]
            # the previous layer's output is torch.split views of one token buffer: take it whole, no 31 MB torch.cat
            qc = _whole(query, split)
            q = (qc if qc is not None else torch.cat(query, dim=1))[0]
            out = routine(q, q, pos_cat[0], ref_2d[0] if ref_2d.dim() == 5 else ref_2d, [(0, n) for n in split], value,
                          spatial_shapes, level_start_index, tpv_levels, reference_points_cams, tpv_vis)
            return torch.split(out[None], split, 1)
        norm_i = attn_i = ffn_i = 0
        identity = query
        for op in self.operation_order:
            if op == 'self_attn':
                q = torch.cat(query, dim=1)
                idt = (q if identity is query else torch.cat(identity, dim=1)) if self.pre_norm else None
                query = torch.split(self.attentions[attn_i](q, q, q, idt, query_pos=pos_cat, reference_points=ref_2d,
                                                            spatial_shapes=tpv_levels[0], level_start_index=tpv_levels[1],
                                                            **kwargs), split, 1)
                attn_i += 1
                identity = query
            elif op == 'norm':
                q = torch.cat(query, dim=1)
                ln = self.norms[norm_i]
                if q.is_cuda and q.dtype == torch.float32 and q.shape[-1] <= 256 and not _needs_grad(q, ln.weight):
                    q = ops.layer_norm(q.contiguous(), ln.weight.detach(), ln.bias.detach(), ln.eps)
                else:
                    q = ln(q)
                query = torch.split(q, split, 1)
                norm_i += 1
            elif op == 'cross_attn':
                query = self.attentions[attn_i](query, key, value, identity if self.pre_norm else None,
                                                spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                                                reference_points_cams=reference_points_cams, tpv_masks=tpv_masks, **kwargs)
                attn_i += 1
                identity = query
            elif op == 'ffn':
                q = torch.cat(query, dim=1)
                idt = (q if identity is query else torch.cat(identity, dim=1)) if self.pre_norm else None
                query = torch.split(self.ffns[ffn_i](q, idt), split, 1)
                ffn_i += 1
        return query

    def _row_routine(self, q, value, kwargs):
        """The routine forward runs on all rows at batch 1 in CUDA fp32, batch_first, post-norm order, no mask:
        forward_rows for inference (eval, no autograd), forward_rows_train otherwise.  None: the op-order loop."""
        if q.shape[0] != 1 or not _cuda_fp32(q, value) or not self.batch_first \
                or tuple(self.operation_order) != POST_NORM_ORDER or kwargs.get('key_padding_mask') is not None:
            return None
        return self.forward_rows if not self.training and not torch.is_grad_enabled() else self.forward_rows_train

    def forward_rows(self, q, q_full, pos, ref, slices, value, spatial_shapes, level_start_index, tpv_levels, uvs, vises):
        """The layer's inference (eval, no autograd, bs = 1, POST_NORM_ORDER) on a set of token rows.
        q [n, C]: the rows, each plane's contiguous slice in hw | zh | wz order, ``slices`` [(begin, count)] per plane;
        q_full [Q, C]: all tokens, the self-attention's value; pos [n, C] / ref [n, 3, P, 2]: the rows' positional embedding and
        cross-view reference points; value [N, sum(hw), 1, C]: the frame's flattened image features with their level tables;
        tpv_levels: the (spatial_shapes, level_start_index) of the three planes; uvs [N, 1, Q_i, D, 2] / vises [N, Q_i]: each
        whole plane's camera projections.  Returns the updated rows [n, C].  Every LayerNorm is folded into the GEMM before it.
        Rows are independent, so any split of the tokens over calls gives bit-identical rows (``dist.ShardedLifter``)."""
        sa, ca, ffn = self.attentions[0], self.attentions[1], self.ffns[0]
        # self-attention (cross_view_hybrid_attention.py:63-124): value = all tokens, queries = these rows (+ pos)
        v = fast_linear(sa.value_proj, q_full)
        qp = q + pos
        offs, logits = _offsets_logits(sa, qp)
        out = ops.tpv_self_attn_forward_rows(v, sa.num_heads, v.shape[1] // sa.num_heads, tpv_levels[0], tpv_levels[1],
                                             offs, logits, ref.contiguous(), sa.num_levels, sa.num_points)
        q = fast_linear(sa.output_proj, out, residual=q, ln=self.norms[0])
        # image cross-attention, one plane at a time (tpvformer/attention/image_cross_attention.py:83-93); the three planes
        # project the same image features with their own value_proj: one GEMM, three column slices
        feat = value[:, :, 0].reshape(-1, value.shape[-1])
        vps = [a.deformable_attention.value_proj for a in ca.attns]
        vrows = fast_linear_cat(ca, '_so_value3', vps, feat)[1] if _fusable(vps, feat) else None
        x = q.new_empty(q.shape)                      # each plane's output_proj writes its own row range: no torch.cat
        o0 = 0
        for i, (b, c) in enumerate(slices):
            if c == 0:
                continue
            att = ca.attns[i]
            da = att.deformable_attention
            qi = q[o0:o0 + c]
            v = vrows[i] if vrows is not None else fast_linear(da.value_proj, feat)
            offs, logits = _offsets_logits(da, qi)
            slots = ops.tpv_cross_attn_forward_rows(v, value.shape[0], da.num_heads, qi.shape[1] // da.num_heads, spatial_shapes,
                                                    level_start_index, offs, logits, uvs[i][:, 0, b:b + c].contiguous(),
                                                    vises[i][:, b:b + c].contiguous(), da.num_levels, da.num_points)
            fast_linear(att.output_proj, slots, residual=qi, out=x[o0:o0 + c], ln=self.norms[1])
            o0 += c
        # FFN on [1, n, C]: the layer's forward returns torch.split views of this one token buffer, which the next layer
        # takes whole (`_whole`) instead of concatenating the planes again
        x = x[None]
        h = fast_linear(ffn.layers[0][0], x, relu=True)
        return fast_linear(ffn.layers[1], h, residual=x if ffn.add_identity else None, ln=self.norms[2])[0]

    def forward_rows_train(self, q, q_full, pos, ref, slices, value, spatial_shapes, level_start_index, tpv_levels, uvs, vises):
        """The layer's training forward (autograd or train mode, bs = 1, POST_NORM_ORDER, CUDA fp32) on a set of token rows,
        the autograd twin of forward_rows: all rows for forward, a rank's rows for the query-sharded training step
        (TPVFormerEncoder.query_shard).  The fused attention cores with their backward kernels (ops.TPVSelfAttnFunction,
        ops.TPVCrossAttnFunction), train_linear, nn.LayerNorm.  Arguments as forward_rows; q_full must be the
        autograd-connected full planes.  Any split of the rows computes every row as the call on all rows does.  Each
        dropout draws its mask for the WHOLE tensor (same shape, same order) and applies this set of rows' part of it
        (_row_dropout), so every rank advances the torch RNG exactly as the call on all rows does and a sharded step has
        one well-defined mask."""
        from .dist import local_rows_of
        sa, ca, ffn = self.attentions[0], self.attentions[1], self.ffns[0]
        sizes = [v.shape[1] for v in vises]
        Q, C = q_full.shape
        n = q.shape[0]
        rows = lambda full: local_rows_of(full, sizes, slices)
        # self-attention: value = all tokens, queries = these rows (+ pos); the residual is the rows without pos
        Hd, L, P = sa.num_heads, sa.num_levels, sa.num_points
        v = train_linear(sa.value_proj, q_full).view(Q, Hd, -1)
        qp = q + pos
        offs = train_linear(sa.sampling_offsets, qp).view(n, Hd, L, P, 2)
        logits = train_linear(sa.attention_weights, qp).view(n, Hd, L, P)
        out = ops.TPVSelfAttnFunction.apply(v, tpv_levels[0], tpv_levels[1], offs, logits, ref)
        # no name holds a [rows, C] tensor that backward does not keep (a projection before its dropout, a dropout before its
        # residual): the forward's peak is what backward saves plus one step's temporaries
        q = self.norms[0](_row_dropout(sa.dropout, train_linear(sa.output_proj, out), (Q, C), rows) + q)
        # image cross-attention, one plane at a time, each on its own rows of q
        n_cam, nv = value.shape[0], value.shape[1]
        feat = value[:, :, 0]
        parts, o0 = [], 0
        for i, (b, c) in enumerate(slices):
            att = ca.attns[i]
            da = att.deformable_attention
            qi = q[o0:o0 + c]
            v = train_linear(da.value_proj, feat).view(n_cam, nv, da.num_heads, -1)
            offs = train_linear(da.sampling_offsets, qi).view(c, da.num_heads, da.num_levels, da.num_points, 2)
            logits = train_linear(da.attention_weights, qi).view(c, da.num_heads, da.num_levels, da.num_points)
            slots = ops.TPVCrossAttnFunction.apply(v, spatial_shapes, level_start_index, offs, logits, uvs[i][:, 0, b:b + c],
                                                   vises[i][:, b:b + c])
            parts.append(_row_dropout(att.dropout, train_linear(att.output_proj, slots), (sizes[i], C),
                                      lambda m, b=b, c=c: m[b:b + c]) + qi)
            o0 += c
        q = self.norms[1](torch.cat(parts, 0))
        # FFN (mmcv FFN: Linear, ReLU, Dropout, Linear, Dropout, + identity)
        l0 = ffn.layers[0]
        h = F.relu(train_linear(l0[0], q))
        h = _row_dropout(l0[2], h, (Q, h.shape[1]), rows)
        out = _row_dropout(ffn.layers[2], train_linear(ffn.layers[1], h), (Q, C), rows)
        if ffn.add_identity:
            out = q + out
        # normed as [1, n, C]: the layer's forward returns torch.split views of this one token buffer, which the next layer
        # takes whole (`_whole`) instead of concatenating the planes again
        return self.norms[2](out[None])[0]


def _row_dropout(drop, x, full_shape, rows):
    """nn.Dropout ``drop`` on the rows ``x`` of a tensor of shape ``full_shape``.  When ``x`` is the whole tensor this is
    ``drop(x)``.  Otherwise the mask is drawn for the whole tensor with the op nn.Dropout runs on a CUDA tensor
    (aten.native_dropout), so the RNG advances as for the whole tensor, and ``rows(mask)`` picks the part that belongs to
    ``x``; x * scale * mask is what native_dropout computes."""
    if tuple(x.shape) == tuple(full_shape):
        return drop(x)
    p = drop.p
    if not drop.training or p == 0:
        return x
    if p == 1:
        return x * 0
    mask = torch.ops.aten.native_dropout(torch.empty(full_shape, device=x.device, dtype=x.dtype), p, True)[1]
    return x * (rows(mask) * (1.0 / (1.0 - p)))


@MODELS.register_module()
class TPVFormerEncoder(nn.Module):
    """A2/A3.  tpvformer_encoder.py:19-290."""

    def __init__(self, mapping_args, embed_dims=128, num_cams=6, num_feature_levels=4, positional_encoding=None,
                 num_points_cross=[64, 64, 8], num_points_self=[16, 16, 16], transformerlayers=None, num_layers=None,
                 camera_aware=False, camera_aware_mid_channels=None, init_cfg=None, **kwargs):
        super().__init__()
        if camera_aware:
            raise NotImplementedError('camera_aware=True (CameraAwareSE) is disabled in every shipped config')
        self.embed_dims, self.num_feature_levels, self.num_cams, self.camera_aware = embed_dims, num_feature_levels, num_cams, False
        self.mapping = GridMeterMapping(**mapping_args)
        H, W, Z = self.mapping.size_h, self.mapping.size_w, self.mapping.size_d
        self.tpv_size = [H, W, Z]
        f = lambda n: torch.arange(n, dtype=torch.float)
        zeros = torch.zeros
        # plane cell centres in metres (tpvformer_encoder.py:84-101)
        hw = self.mapping.grid2meter(torch.stack([f(H)[:, None].expand(H, W), f(W)[None].expand(H, W), zeros(H, W)], -1))[..., [0, 1]]
        zh = self.mapping.grid2meter(torch.stack([f(H)[None].expand(Z, H), zeros(Z, H), f(Z)[:, None].expand(Z, H)], -1))[..., [1, 2]]
        wz = self.mapping.grid2meter(torch.stack([zeros(W, Z), f(W)[:, None].expand(W, Z), f(Z)[None].expand(W, Z)], -1))[..., [0, 2]]
        pe = dict(positional_encoding)
        pe['tpv_meters'] = [hw, zh, wz]
        self.positional_encoding = build_positional_encoding(pe)
        if isinstance(transformerlayers, dict):
            transformerlayers = [copy.deepcopy(transformerlayers) for _ in range(num_layers)]
        assert isinstance(transformerlayers, (list, tuple)) and len(transformerlayers) == num_layers
        self.num_layers = num_layers
        self.layers = nn.ModuleList([build_transformer_layer(copy.deepcopy(c)) for c in transformerlayers])
        self.pre_norm = self.layers[0].pre_norm
        self.level_embeds = nn.Parameter(torch.randn(num_feature_levels, embed_dims))
        self.cams_embeds = nn.Parameter(torch.randn(num_cams, embed_dims))
        self.num_points_cross, self.num_points_self = num_points_cross, num_points_self
        r_hw, r_zh, r_wz = _pillar_tables(self.mapping, num_points_cross)
        self.register_buffer('ref_3d_hw', r_hw, False)
        self.register_buffer('ref_3d_zh', r_zh, False)
        self.register_buffer('ref_3d_wz', r_wz, False)
        assert num_points_self[0] == num_points_self[1] == num_points_self[2]
        self.register_buffer('cross_view_ref_points', _cross_view_refs(H, W, Z, num_points_self[0]), False)
        self.register_buffer('tpv_spatial_shapes', torch.tensor([[H, W], [Z, H], [W, Z]], dtype=torch.int64), False)
        self.register_buffer('tpv_level_start', torch.tensor([0, H * W, H * W + Z * H], dtype=torch.int64), False)
        # query-sharded training (forward_query_sharded): (rank, world) of this process, and the process group of the
        # exchange (None: the default group)
        self.query_shard = None
        self.query_shard_group = None

    def init_weights(self):
        """tpvformer_encoder.py:174-190."""
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, (BEVCrossAttention,)):
                m.init_weight()
            elif isinstance(m, (BEVDeformableAttention, CrossViewHybridAttention)):
                m.init_weights()
        nn.init.normal_(self.level_embeds)
        nn.init.normal_(self.cams_embeds)

    def project_reference_points(self, metas, device):
        """A4: three point_sampling calls (tpvformer_encoder.py:205-210) -> per plane uv [N,B,Q,D,2],
        mask [N,B,Q,D] uint8, vis [N,Q] uint8.  B must be 1 (as everywhere in the reference head).  Frames from the
        reference's data wrapper carry metas[0]['focal_ratios_x' / '_y'] (RandomScaleImageMultiViewImage): uv is rescaled
        per camera after the frustum test (bevformer/utils.py:198-204), see _focal_scale."""
        if 'img_augmentation' in metas[0]:
            raise NotImplementedError("the post_rots / post_trans branch of point_sampling (metas['img_augmentation']) is not "
                                      'implemented: no shipped data pipeline produces it')
        l2i = _metas_matrix(metas, 'lidar2img', device)
        assert l2i.shape[0] == 1, 'only bs = 1 is supported (the reference head asserts the same)'
        scale_xy = _focal_scale(metas, l2i.shape[1], device)
        shp = metas[0]['img_shape']
        uvs, masks, vises = [], [], []
        for ref in (self.ref_3d_hw, self.ref_3d_zh, self.ref_3d_wz):
            uv, mask, vis = ops.point_sampling(ref, l2i[0].contiguous(), (shp[0], shp[1]), scale_xy)
            uvs.append(uv[:, None])
            masks.append(mask[:, None])
            vises.append(vis)
        return uvs, masks, vises

    def forward_layers(self, tpv_query, key, value, tpv_pos=None, spatial_shapes=None, level_start_index=None,
                       img_metas=None, **kwargs):
        dev = tpv_query[0].device
        uvs, masks, vises = self.project_reference_points(img_metas, dev)
        bs = tpv_query[0].shape[0]
        ref_cross_view = self.cross_view_ref_points[None].expand(bs, -1, -1, -1, -1)
        for layer in self.layers:
            tpv_query = layer(tpv_query, key, value, tpv_pos=tpv_pos, ref_2d=ref_cross_view, spatial_shapes=spatial_shapes,
                              level_start_index=level_start_index, reference_points_cams=uvs, tpv_masks=masks,
                              tpv_size=self.tpv_size, tpv_vis=vises,
                              tpv_levels=(self.tpv_spatial_shapes, self.tpv_level_start), **kwargs)
        return tpv_query

    def flatten_features(self, img_feats):
        """A3: [B,N,C,h,w] x L -> [N, sum(hw), B, C] with camera + level embeddings (tpvformer_encoder.py:261-277)."""
        f0 = img_feats[0]
        if f0.is_cuda and f0.dtype == torch.float32 and f0.shape[0] == 1 and all(f.is_contiguous() for f in img_feats) \
                and not _needs_grad(self.cams_embeds, *img_feats):
            shapes = tuple((f.shape[3], f.shape[4]) for f in img_feats)  # fused transposing pass (so_flatten_level)
            key = (shapes, f0.device)
            if getattr(self, '_shape_key', None) != key:                 # the two tiny int64 tables are per-resolution constants
                spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=f0.device)
                level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
                self._shape_key, self._shape_val = key, (spatial_shapes, level_start_index)
            spatial_shapes, level_start_index = self._shape_val
            return ops.flatten_levels(img_feats, self.cams_embeds.detach().contiguous(), self.level_embeds.detach().contiguous()), \
                spatial_shapes, level_start_index
        feats, shapes = [], []
        for lvl, feat in enumerate(img_feats):
            bs, num_cam, c, h, w = feat.shape
            shapes.append((h, w))
            f = feat.flatten(3).permute(1, 0, 3, 2)
            feats.append(f + self.cams_embeds[:, None, None, :] + self.level_embeds[None, None, lvl:lvl + 1, :])
        dev = img_feats[0].device
        spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=dev)
        level_start_index = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
        return torch.cat(feats, 2).permute(0, 2, 1, 3).contiguous(), spatial_shapes, level_start_index

    def _tpv_pos(self):
        """Positional embeddings depend on the weights only: recomputed per call under autograd (training), cached per
        parameter version otherwise (tpvformer_encoder.py:254 recomputes them every frame)."""
        pe = self.positional_encoding
        ws = [pe.position_layer_hw.weight, pe.position_layer_zh.weight, pe.position_layer_wz.weight,
              pe.position_layer_hw.bias, pe.position_layer_zh.bias, pe.position_layer_wz.bias]
        if torch.is_grad_enabled() and any(w.requires_grad for w in ws):
            return pe()
        key = tuple((w._version, w.data_ptr()) for w in ws)
        if getattr(self, '_pos_key', None) != key:
            with torch.no_grad():
                vals = pe()
                self._pos_key, self._pos_val = key, vals
                self._pos_cat = torch.cat(vals, 0).unsqueeze(0)      # [1, Q_hw + Q_zh + Q_wz, C]: what every layer concatenates
        return self._pos_val

    def frame_inputs(self, ms_img_feats):
        """The per-frame inputs every layer reads besides the camera projections (``project_reference_points``):
        (tpv_pos, feat_flatten, spatial_shapes, level_start_index).  tpv_pos is the cached [1, Q_hw + Q_zh + Q_wz, C]
        concatenation at bs = 1 without autograd (the layers accept a tensor: no 31 MB cat per layer), else the per-plane list."""
        bs = ms_img_feats[0].shape[0]
        pos = self._tpv_pos()
        if bs == 1 and getattr(self, '_pos_val', None) is pos:
            tpv_pos = self._pos_cat
        else:
            tpv_pos = [p.unsqueeze(0).repeat(bs, 1, 1) if bs > 1 else p.unsqueeze(0) for p in pos]
        return (tpv_pos,) + self.flatten_features(ms_img_feats)

    # ---- query-sharded training (query_shard = (rank, world)): each rank runs every layer on its own rows of each plane
    def shard_state(self, ms_img_feats, metas):
        """The per-frame inputs every rank of a query-sharded training step computes whole (under autograd): positional
        embeddings [Q_total, C], flattened image features with their level tables, camera projections of every plane."""
        tpv_pos, feat, shapes, lsi = self.frame_inputs(ms_img_feats)
        pos = torch.cat([p[0] for p in tpv_pos], 0) if isinstance(tpv_pos, (list, tuple)) else tpv_pos[0]
        uvs, _, vises = self.project_reference_points(metas, feat.device)
        return dict(pos=pos, feat=feat, shapes=shapes, lsi=lsi, uvs=uvs, vises=vises)

    def shard_layer(self, li, qfull, st, rank, world):
        """Layer li of the query-sharded training step: the full planes qfull [Q_total, C] (autograd-connected) -> this
        rank's updated rows (dist.plane_slices of each plane, plane after plane)."""
        from .dist import local_rows, plane_slices
        H, W, Z = self.tpv_size
        sizes = [H * W, Z * H, W * Z]
        rows = lambda t: local_rows(t, sizes, rank, world)
        return self.layers[li].forward_rows_train(
            rows(qfull), qfull, rows(st['pos']), rows(self.cross_view_ref_points), plane_slices(sizes, rank, world), st['feat'],
            st['shapes'], st['lsi'], (self.tpv_spatial_shapes, self.tpv_level_start), st['uvs'], st['vises'])

    def forward_query_sharded(self, representation, ms_img_feats, metas, rank, world, collective=None, reduce_scatter=None,
                              group=None):
        """The encoder's training forward with the queries sharded over ``world`` ranks: the shared set-up (shard_state),
        then per layer this rank's rows (shard_layer) and ONE dist.all_gather_rows that rebuilds the planes (its backward
        is one reduce-scatter).  Returns the full planes [1, Q_i, C] x 3 on every rank; the rows equal the unsharded
        training forward's.  ``collective`` / ``reduce_scatter`` / ``group``: as dist.all_gather_rows."""
        from .dist import all_gather_rows
        H, W, Z = self.tpv_size
        sizes = [H * W, Z * H, W * Z]
        if min(sizes) < world:
            raise ValueError('query_shard: a plane of %s rows cannot be split over %d ranks (a rank without rows would leave '
                             'parameters without a gradient)' % (sizes, world))
        if representation[0].shape[0] != 1 or not _cuda_fp32(representation[0], ms_img_feats[0]):
            raise NotImplementedError('query_shard: batch 1, CUDA fp32 only')
        for layer in self.layers:
            if tuple(layer.operation_order) != POST_NORM_ORDER or not layer.batch_first:
                raise NotImplementedError('query_shard: operation_order %r' % (layer.operation_order,))
        st = self.shard_state(ms_img_feats, metas)
        qfull = torch.cat([p[0] for p in representation], 0)
        for li in range(len(self.layers)):
            local = self.shard_layer(li, qfull, st, rank, world)
            qfull = all_gather_rows(local, sizes, rank, world, collective, reduce_scatter, group)
        return [t[None] for t in torch.split(qfull, sizes, 0)]

    def forward(self, representation, ms_img_feats=None, metas=None, **kwargs):
        shard = getattr(self, 'query_shard', None)
        if shard is not None and shard[1] > 1 and self.training and torch.is_grad_enabled():
            return {'representation': self.forward_query_sharded(representation, ms_img_feats, metas, shard[0], shard[1],
                                                                 group=getattr(self, 'query_shard_group', None))}
        tpv_pos, feat_flatten, spatial_shapes, level_start_index = self.frame_inputs(ms_img_feats)
        tpv_embed = self.forward_layers(representation, feat_flatten, feat_flatten, tpv_pos=tpv_pos,
                                        spatial_shapes=spatial_shapes, level_start_index=level_start_index, img_metas=metas)
        return {'representation': list(tpv_embed)}
