"""Generate tests/golden/reference_golden_focal.npz: the reference's point_sampling with the focal-ratio metas.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_focal.py <path to the SelfOcc checkout>
model/encoder/bevformer/utils.py is loaded by file path and ``point_sampling`` (utils.py:116-206) is executed UNMODIFIED
with the focal_ratios_x / _y that RandomScaleImageMultiViewImage (dataset/transform_3d.py:350-363) writes, at the ratios
the shipped configs produce: kitti_raw_depth (scale_rate 0.84, pad_scale_rate [0.8649, 0.8421]) and kitti_novel_depth
(pad_scale_rate [1.038, 1.0]) on one camera, nuScenes (scale_rate 0.5: exactly 1.0) on six, and six per-camera ratios
around 1 (the random_scale option) that push visible samples outside [0, 1].  Inputs are seeded and stored beside the
outputs.
"""
import importlib.util
import os
import sys
import numpy as np
import torch

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))


def load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rig(K, yaws, t):
    """lidar2img [N, 4, 4] of cameras at ``t`` yawed by ``yaws`` (degrees), built as make_golden.py's point_sampling rig."""
    l2i = []
    for yaw in yaws:
        a = np.deg2rad(yaw)
        c2l = np.eye(4)
        # camera axes (x right, y down, z forward) expressed in the lidar frame (x right, y fwd, z up)
        fwd = np.array([np.sin(-a), np.cos(-a), 0.])
        right = np.array([np.cos(-a), -np.sin(-a), 0.])
        down = np.array([0., 0., -1.])
        c2l[:3, 0], c2l[:3, 1], c2l[:3, 2], c2l[:3, 3] = right, down, fwd, t
        l2i.append(K @ np.linalg.inv(c2l))
    return np.stack(l2i)


def main():
    bu = load('model/encoder/bevformer/utils.py', 'ref_bev_utils')
    torch.manual_seed(5)
    k_kitti = np.array([[721.5, 0, 609.6, 0], [0, 721.5, 172.9, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    k_nusc = np.array([[1266., 0, 800, 0], [0, 1266., 450, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    kitti_l2i, kitti_img = rig(k_kitti, (0.,), [0., 0., 1.7]), (370, 1226)
    nusc_l2i, nusc_img = rig(k_nusc, (0., -55., 55., 180., -110., 110.), [0.3, 0.5, 1.5]), (900, 1600)
    kitti_pts = lambda: torch.rand(1, 4, 160, 3) * torch.tensor([50., 50., 6.4]) - torch.tensor([25., 0., 2.])
    nusc_pts = lambda: (torch.rand(1, 4, 160, 3) - 0.5) * torch.tensor([80., 80., 8.])
    cases = {
        # name: (lidar2img [N,4,4], img_shape, ratios_x, ratios_y, points)  -- ratios as the transform computes them
        'kitti_raw': (kitti_l2i, kitti_img, [0.84 / 0.8421], [0.84 / 0.8649], kitti_pts()),
        'kitti_novel': (kitti_l2i, kitti_img, [1.0 / 1.0], [1.0 / 1.038], kitti_pts()),
        'nusc': (nusc_l2i, nusc_img, [0.5 / 0.5] * 6, [0.5 / 0.5] * 6, nusc_pts()),
        'mixed': (nusc_l2i, nusc_img, [0.91, 1.08, 0.97, 1.05, 1.0, 0.94], [1.06, 0.92, 1.08, 0.99, 1.03, 0.95], nusc_pts()),
    }
    out = {}
    for name, (l2i, img, rx, ry, ref3d) in cases.items():
        metas = [dict(lidar2img=list(l2i), img_shape=img, focal_ratios_x=rx, focal_ratios_y=ry)]
        rc, mk = bu.point_sampling(ref3d, metas)
        out[name + '_ref3d'], out[name + '_lidar2img'] = ref3d.numpy(), l2i[None]
        out[name + '_img_shape'] = np.array(img)
        out[name + '_ratios_x'], out[name + '_ratios_y'] = np.array(rx), np.array(ry)
        out[name + '_uv'], out[name + '_mask'] = rc.numpy(), mk.numpy()
        outside = int(((rc < 0) | (rc > 1)).any(-1)[mk].sum())
        print('%s: %d of %d samples visible, %d of them outside [0, 1]' % (name, int(mk.sum()), mk.numel(), outside))
    np.savez_compressed(os.path.join(HERE, 'reference_golden_focal.npz'), **out)
    print('wrote focal golden:', len(out), 'arrays')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'model', 'encoder', 'bevformer', 'utils.py')):
        sys.exit('usage: python tests/golden/make_golden_focal.py <path to a huang-yh/SelfOcc checkout>')
    main()
