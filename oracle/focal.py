"""Oracle: the focal-ratio branch of point_sampling (test infrastructure, see oracle/__init__.py).

bevformer/utils.py:198-204: when metas[0] carries ``focal_ratios_x`` / ``focal_ratios_y`` (RandomScaleImageMultiViewImage,
dataset/transform_3d.py:362-363, inserted by the data wrapper of every nuScenes config and of kitti_raw_depth /
kitti_novel_depth), the projected uv is multiplied per camera by the ratios AFTER the frustum mask is computed.
Pinned by tests/golden/reference_golden_focal.npz (tests/golden/make_golden_focal.py).

The pieces of ``oracle.lifting`` are looked up on that module at call time, so a test that promotes them to fp64 by
replacing them there (tests/test_gpu_encoder_parity.py) promotes them here too.
"""
import torch

from . import lifting


def focal_scale_ref(uv, ratios_x, ratios_y):
    """uv [N, B, Q, D, 2] from point_sampling_ref -> uv with x times ratios_x[cam] and y times ratios_y[cam]; the mask of
    point_sampling_ref is left as it is (it is computed first, from the unscaled uv).  The ratios are metas[0]'s lists,
    rounded to fp32 by ``new_tensor`` and broadcast per camera by ``view(-1, 1, 1, 1, 1)`` (length 1 or N)."""
    sx = torch.tensor(ratios_x, dtype=torch.float32).view(-1, 1, 1, 1, 1).to(uv.dtype)
    sy = torch.tensor(ratios_y, dtype=torch.float32).view(-1, 1, 1, 1, 1).to(uv.dtype)
    uv = uv.clone()
    uv[..., :1] = uv[..., :1] * sx
    uv[..., 1:] = uv[..., 1:] * sy
    return uv


def tpv_encoder_ref(p, mapping, planes, ms_img_feats, lidar2img, img_shape, cfg, focal_ratios):
    """lifting.tpv_encoder_ref (TPVFormerEncoder.forward, tpvformer_encoder.py:192-290) on a frame whose metas carry
    focal_ratios = (metas[0]['focal_ratios_x'], metas[0]['focal_ratios_y']): every plane's camera projection goes through
    focal_scale_ref after point_sampling_ref, as point_sampling does in the reference."""
    B = planes[0].shape[0]
    H, W, Z = mapping.size_h, mapping.size_w, mapping.size_d
    feats = lifting.tpv_pos_features(mapping, cfg['num_freqs'], cfg['tot_range'])
    tpv_pos = [lifting._lin(p, 'positional_encoding.position_layer_' + n, f)[None].repeat(B, 1, 1)
               for n, f in zip(('hw', 'zh', 'wz'), feats)]
    feat, shapes = lifting.flatten_img_feats(p, ms_img_feats)
    ref_cams, masks = [], []
    for r3 in lifting.ref_3d_tables(mapping, cfg['num_points_cross']):
        rc, m = lifting.point_sampling_ref(r3[None].repeat(B, 1, 1, 1), lidar2img, img_shape)
        ref_cams.append(focal_scale_ref(rc, *focal_ratios))
        masks.append(m)
    ref_2d = lifting.cross_view_ref_points(H, W, Z, [cfg['num_points_self']] * 3)[None].expand(B, -1, -1, -1, -1)
    for i in range(cfg['num_layers']):
        planes = lifting.tpv_layer_ref(p, 'layers.%d.' % i, planes, tpv_pos, feat, shapes, ref_2d, ref_cams, masks,
                                       (H, W, Z), cfg)
    return planes
