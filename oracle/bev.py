"""Oracle: the BEV-only model (config/nuscenes/nuscenes_occ_bev.py; test infrastructure, see oracle/__init__.py).

Restated from the reference (file:line in each docstring), fp64-capable (every function follows its inputs' dtype), on the
building blocks of oracle/lifting.py.  Pinned by tests/golden/reference_golden_bev.npz (make_golden_bev.py runs the
reference's modules).  Two details of the reference are reproduced as they are, not "fixed":

* the self-attention's reference point of query (h, w) is (h / (H - 1), w / (W - 1)) handed to mmcv as (x, y) over
  spatial_shapes [[H, W]] (bevformer_encoder.py:114-117,151-152, bevformer_encoder_layer.py:168-180), while the value is the
  query plane in h * W + w order: x, derived from h, indexes the column (w) axis, so query (h, w) samples around the
  transposed cell, with the (H - 1) vs W normaliser and align_corners=False's -0.5;
* the decode's column j of a BEV cell is voxel z = j // Cf, channel c = j % Cf (reshape(..., Z, -1), bev_nerf.py:78-80).
"""
import torch
import torch.nn.functional as F

from .focal import focal_scale_ref
from .lifting import (_lin, _ln, ffn_ref, flatten_img_feats, image_cross_attn_ref, msda_ref, point_sampling_ref,
                      pos_freq_features)


def bev_grid(H, W, dtype=torch.float):
    """bevformer_encoder.py:72-74: [H, W, (h, w)] cell indices."""
    return torch.stack([torch.arange(H, dtype=dtype)[:, None].expand(-1, W), torch.arange(W, dtype=dtype)[None].expand(H, -1)], -1)


def bev_pos_features(mapping, num_freqs, tot_range):
    """bevformer_pos_embed.py:14-28: cell metres normalised by the point-cloud range, then sin / cos -> [H*W, 4 num_freqs]."""
    r = tot_range if isinstance(tot_range, (list, tuple)) else [-1.0 * tot_range, -1.0 * tot_range, 0., tot_range, tot_range, 0.]
    m = mapping.grid2meter(bev_grid(mapping.size_h, mapping.size_w)).clone()
    m[..., 0] = (m[..., 0] - r[0]) / (r[3] - r[0])
    m[..., 1] = (m[..., 1] - r[1]) / (r[4] - r[1])
    return pos_freq_features(num_freqs, m)


def bev_ref_tables(mapping, num_points_cross):
    """bevformer_encoder.py:106-117 -> (ref_3d [D, H*W, 3] metres of each cell's pillar, ref_2d [H, W, 2])."""
    H, W, Z = mapping.size_h, mapping.size_w, mapping.size_d
    g = bev_grid(H, W)
    d = torch.linspace(0, Z - 1, num_points_cross)
    g3 = torch.cat([g[:, :, None].expand(-1, -1, num_points_cross, -1), d.reshape(1, 1, -1, 1).expand(H, W, -1, -1)], -1)
    ref_3d = mapping.grid2meter(g3).flatten(0, 1).transpose(0, 1).contiguous()
    ref_2d = g.clone()
    ref_2d[..., 0] = ref_2d[..., 0] / (H - 1)
    ref_2d[..., 1] = ref_2d[..., 1] / (W - 1)
    return ref_3d, ref_2d


def bev_self_attn_ref(p, pre, query, query_pos, ref_2d, bev_size, num_heads, num_points):
    """mmcv MultiScaleDeformableAttention.forward as the BEV layer calls it (bevformer_encoder_layer.py:168-180): value =
    query (no pos), identity = query, reference_points ref_2d [B, H*W, 1, 2] broadcast over the points, spatial_shapes
    [[H, W]], eval mode."""
    B, Q, C = query.shape
    ss = [tuple(bev_size)]
    q = query + query_pos
    value = _lin(p, pre + 'value_proj', query).view(B, Q, num_heads, -1)
    off = _lin(p, pre + 'sampling_offsets', q).view(B, Q, num_heads, 1, num_points, 2)
    aw = _lin(p, pre + 'attention_weights', q).view(B, Q, num_heads, num_points).softmax(-1).view(B, Q, num_heads, 1, num_points)
    norm = torch.tensor([[float(bev_size[1]), float(bev_size[0])]], dtype=off.dtype)
    loc = ref_2d[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    return _lin(p, pre + 'output_proj', msda_ref(value, ss, loc, aw)) + query


def bev_layer_ref(p, pre, query, bev_pos, feat, img_shapes, ref_2d, ref_cam, mask, bev_size, cfg):
    """BEVFormerLayer.forward (bevformer_encoder_layer.py:121-216), operation_order ('self_attn', 'norm', 'cross_attn',
    'norm', 'ffn', 'norm'), eval mode.  query [B, H*W, C]; ref_cam [N, B, H*W, D, 2]; mask [N, B, H*W, D]."""
    q = bev_self_attn_ref(p, pre + 'attentions.0.', query, bev_pos, ref_2d, bev_size, cfg['num_heads'], cfg['num_points_self'])
    q = _ln(p, pre + 'norms.0', q)
    q = image_cross_attn_ref(p, pre + 'attentions.1.', q, feat, img_shapes, ref_cam, mask, cfg['num_heads'], cfg['num_cams'])[0]
    q = _ln(p, pre + 'norms.1', q)
    return _ln(p, pre + 'norms.2', ffn_ref(p, pre + 'ffns.0.', q))


def bev_encoder_ref(p, mapping, bev, ms_img_feats, lidar2img, img_shape, cfg, focal_ratios=None):
    """BEVFormerEncoder.forward (bevformer_encoder.py:135-223), eval mode.  bev [B, H*W, C] -> [B, H*W, C].  cfg: num_freqs,
    tot_range, num_points_cross, num_points_self, num_heads, num_cams, num_layers.  focal_ratios: (metas[0]['focal_ratios_x'],
    ['focal_ratios_y']) of a frame that carries them (oracle/focal.py)."""
    B = bev.shape[0]
    H, W = mapping.size_h, mapping.size_w
    dt = bev.dtype
    pos = _lin(p, 'positional_encoding.position_layer', bev_pos_features(mapping, cfg['num_freqs'], cfg['tot_range']).to(dt))
    feat, shapes = flatten_img_feats(p, ms_img_feats)
    ref_3d, ref_2d = bev_ref_tables(mapping, cfg['num_points_cross'])
    ref_cam, mask = point_sampling_ref(ref_3d[None].repeat(B, 1, 1, 1), lidar2img, img_shape)
    if focal_ratios is not None:
        ref_cam = focal_scale_ref(ref_cam, *focal_ratios)
    ref_2d = ref_2d.to(dt).reshape(1, -1, 1, 2).repeat(B, 1, 1, 1)
    q = bev
    for i in range(cfg['num_layers']):
        q = bev_layer_ref(p, 'layers.%d.' % i, q, pos[None].repeat(B, 1, 1), feat, shapes, ref_2d, ref_cam.to(dt), mask,
                          (H, W), cfg)
    return q


def bev_decode_ref(bev, sizes, w1, b1, w2, b2, row_chunk=8192):
    """bev_nerf.py:74-81 (tpv=False, density_layers=2): bev [H*W, C] -> decoded volume [Cf, H, W, Z] (the layout of
    oracle/render.py:tpv_decode_ref), column j of a cell = voxel j // Cf, channel j % Cf."""
    H, W, Z = sizes
    out = []
    for r0 in range(0, bev.shape[0], row_chunk):
        f = F.linear(F.softplus(F.linear(F.softplus(bev[r0:r0 + row_chunk]), w1, b1)), w2, b2)
        out.append(f)
    return torch.cat(out, 0).reshape(H, W, Z, -1).permute(3, 0, 1, 2).contiguous()
