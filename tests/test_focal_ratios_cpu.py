"""CPU: the focal-ratio rescale of point_sampling (bevformer/utils.py:198-204), which every frame of the nuScenes and the two
depth KITTI configs carries (RandomScaleImageMultiViewImage writes metas['focal_ratios_x' / '_y']).

* the oracle (point_sampling_ref + focal_scale_ref) against the reference's own point_sampling, run unmodified on the
  shipped configs' ratios (tests/golden/reference_golden_focal.npz, tests/golden/make_golden_focal.py), bit for bit;
* the C ABI entry point so_point_sampling_scaled refuses what so_point_sampling refuses, before any CUDA call;
* TPVFormerEncoder.project_reference_points reads the ratios of metas shaped like the reference's data wrapper output and
  raises ValueError for malformed ones before any launch."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from selfocc_b200 import configs, synth
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401  registers the modules

HERE = os.path.dirname(os.path.abspath(__file__))
T = lambda a: torch.from_numpy(np.asarray(a))

# The ratios RandomScaleImageMultiViewImage writes (dataset/transform_3d.py:341-363) for each shipped config that inserts
# it (dataset_wrapper_temporal.py:59-61): scale / pad_scale_rate[1] for x, scale / pad_scale_rate[0] for y, the pad rate
# defaulting to the scale.  kitti_occ (scale 1, no pad rate) writes none.
WRAPPER_RATIOS = {
    'nuscenes/nuscenes_occ.py': (6, 0.5, [0.5, 0.5]),
    'nuscenes/nuscenes_depth.py': (6, 0.5, [0.5, 0.5]),
    'nuscenes/nuscenes_novel_depth.py': (6, 0.5, [0.5, 0.5]),
    'kitti_raw/kitti_raw_depth.py': (1, 0.84, [0.8649, 0.8421]),
    'kitti/kitti_novel_depth.py': (1, 1.0, [1.038, 1.0]),
}


def wrapper_metas(n_cam, scale_rate, pad_scale_rate, img_shape):
    """metas[0] with the keys dataset_wrapper_temporal.py:93-117 emits (the head's matrices aside)."""
    l2i, _ = synth.camera_rig(synth.NUSC_YAWS[:n_cam], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    scales = [scale_rate] * n_cam
    return dict(lidar2img=list(l2i), img_shape=tuple(img_shape), scale_rate=scale_rate,
                focal_ratios_x=[s / pad_scale_rate[1] for s in scales], focal_ratios_y=[s / pad_scale_rate[0] for s in scales],
                flip=False)


# --------------------------------------------------------------------------------------------- oracle vs the reference
@pytest.mark.parametrize('case', ['kitti_raw', 'kitti_novel', 'nusc', 'mixed'])
def test_focal_scale_oracle_matches_reference_point_sampling(case):
    from oracle import lifting as ol
    from oracle.focal import focal_scale_ref
    g = np.load(os.path.join(HERE, 'golden', 'reference_golden_focal.npz'))
    k = lambda n: g['%s_%s' % (case, n)]
    rx, ry = k('ratios_x').tolist(), k('ratios_y').tolist()
    uv0, mask = ol.point_sampling_ref(T(k('ref3d')), T(k('lidar2img')), tuple(int(v) for v in k('img_shape')))
    uv = focal_scale_ref(uv0, rx, ry)
    assert torch.equal(mask, T(k('mask'))) and torch.equal(uv, T(k('uv')))
    assert 0 < mask.sum() < mask.numel()
    outside = int(((uv < 0) | (uv > 1)).any(-1)[mask].sum())
    if case == 'nusc':
        assert rx == ry == [1.0] * 6 and torch.equal(uv, uv0)             # scale_rate / pad rate: exactly 1.0
    elif case == 'mixed':
        assert min(rx + ry) < 1 < max(rx + ry) and outside > 0             # visible samples outside [0, 1]
    else:
        assert len(rx) == 1 and not torch.equal(uv, uv0)


# --------------------------------------------------------------------------------------------- C ABI
def test_scaled_entry_point_rejects_what_the_plain_one_rejects_without_a_gpu():
    """so_point_sampling_scaled returns SO_ERR_INVALID_ARG (-1) before any CUDA call exactly where so_point_sampling does: a
    null required pointer (ref_3d, lidar2img, uv), a size below 1, a non-positive or NaN image size."""
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N = None
    one = C.c_void_p(16)   # non-null, 16-byte aligned dummy (never dereferenced on these paths)
    ok = dict(ref=one, l2i=one, D=1, Q=1, N=1, h=1.0, w=1.0, uv=one)
    bad = [dict(ref=N), dict(l2i=N), dict(uv=N), dict(D=0), dict(Q=0), dict(N=0), dict(D=-3), dict(h=0.0), dict(w=-1.0),
           dict(h=float('nan')), dict(w=float('nan'))]
    for b in bad:
        a = dict(ok, **b)
        plain = lib.so_point_sampling(a['ref'], a['l2i'], a['D'], a['Q'], a['N'], a['h'], a['w'], a['uv'], N, N, N)
        for scale in (N, one):
            scaled = lib.so_point_sampling_scaled(a['ref'], a['l2i'], scale, a['D'], a['Q'], a['N'], a['h'], a['w'], a['uv'],
                                                  N, N, N)
            assert scaled == plain == -1, (b, scale, scaled, plain)


# --------------------------------------------------------------------------------------------- encoder
def _encoder(n_cam):
    margs, rng = synth.small_mapping(6, 3)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=n_cam, num_layers=1, num_points_cross=(5, 5, 3),
                                  num_points_self=4)
    return build_head(cfg['encoder'])


@pytest.mark.parametrize('name', sorted(WRAPPER_RATIOS))
def test_wrapper_ratios_become_one_fp32_pair_per_camera(name):
    """The five shipped configs' ratios, as the wrapper emits them (lists of Python floats) and as numpy arrays or tensors,
    give scale_xy [N, 2]: the values rounded to fp32 as the reference's new_tensor rounds them."""
    from selfocc_b200.encoder import _focal_scale
    n_cam, scale, pad = WRAPPER_RATIOS[name]
    m = wrapper_metas(n_cam, scale, pad, (90, 160))
    want = torch.stack([torch.tensor(np.asarray(m['focal_ratios_x'])).float(), torch.tensor(np.asarray(m['focal_ratios_y'])).float()], -1)
    for conv in (lambda v: v, np.asarray, lambda v: torch.tensor(v, dtype=torch.float64), lambda v: torch.tensor(v).float()):
        got = _focal_scale([dict(m, focal_ratios_x=conv(m['focal_ratios_x']), focal_ratios_y=conv(m['focal_ratios_y']))], n_cam,
                           torch.device('cpu'))
        assert got.dtype == torch.float32 and got.is_contiguous() and torch.equal(got, want)
    assert _focal_scale([dict(lidar2img=m['lidar2img'], img_shape=(90, 160))], n_cam, torch.device('cpu')) is None


def test_one_ratio_broadcasts_over_the_cameras():
    from selfocc_b200.encoder import _focal_scale
    got = _focal_scale([dict(focal_ratios_x=[1.07], focal_ratios_y=np.array([0.96]))], 6, torch.device('cpu'))
    assert got.shape == (6, 2) and torch.equal(got, torch.tensor([[1.07, 0.96]] * 6, dtype=torch.float32))


@pytest.mark.parametrize('bad', ['x_only', 'y_only', 'x_len_2', 'y_len_7', 'x_empty'])
def test_malformed_ratios_raise_value_error_before_any_launch(bad):
    enc = _encoder(6)
    m = wrapper_metas(6, 0.5, [0.5, 0.5], (90, 160))
    if bad == 'x_only':
        del m['focal_ratios_y']
    elif bad == 'y_only':
        del m['focal_ratios_x']
    elif bad == 'x_len_2':
        m['focal_ratios_x'] = [1.0, 1.0]
    elif bad == 'y_len_7':
        m['focal_ratios_y'] = torch.ones(7)
    else:
        m['focal_ratios_x'] = []
    with pytest.raises(ValueError, match='focal_ratios'):
        enc.project_reference_points([m], torch.device('cpu'))


def test_img_augmentation_stays_refused():
    enc = _encoder(6)
    m = dict(wrapper_metas(6, 0.5, [0.5, 0.5], (90, 160)), img_augmentation=dict(post_rots=None, post_trans=None))
    with pytest.raises(NotImplementedError, match='no shipped data pipeline'):
        enc.project_reference_points([m], torch.device('cpu'))
