"""Deterministic synthetic inputs for tests and bench.py (SURVEY.md section 8d): pinhole camera rigs,
analytic SDF scenes, random TPV planes / FPN features.  Pure torch/numpy, device-agnostic."""
import math
import numpy as np
import torch

NUSC_YAWS = (0., -55., 55., 180., 110., -110.)

NUSC_MAPPING = dict(nonlinear_mode='linear', h_size=[128, 0], h_range=[51.2, 0], h_half=False, w_size=[128, 0],
                    w_range=[51.2, 0], w_half=False, d_size=[30, 0], d_range=[-4.0, 5.0, 5.0])
NUSC_RANGE = [-51.2, -51.2, -4.0, 51.2, 51.2, 5.0]


def small_mapping(hw=16, d=8, rng=12.8, z0=-2.0, z1=3.0):
    return dict(nonlinear_mode='linear', h_size=[hw, 0], h_range=[rng, 0], h_half=False, w_size=[hw, 0],
                w_range=[rng, 0], w_half=False, d_size=[d, 0], d_range=[z0, z1, z1]), [-rng, -rng, z0, rng, rng, z1]


def camera_rig(yaws_deg=NUSC_YAWS, f=1266.0, cx=800.0, cy=450.0, height=1.5, radius=0.5):
    """lidar frame: x right, y forward, z up; camera frame: x right, y down, z forward.
    Returns (lidar2img [N,4,4], img2lidar [N,4,4]) float64 numpy."""
    K = np.array([[f, 0, cx, 0], [0, f, cy, 0], [0, 0, 1, 0], [0, 0, 0, 1.]])
    l2i, i2l = [], []
    for yaw in yaws_deg:
        a = np.deg2rad(yaw)
        fwd = np.array([-np.sin(a), np.cos(a), 0.])
        right = np.array([np.cos(a), np.sin(a), 0.])
        down = np.array([0., 0., -1.])
        c2l = np.eye(4)
        c2l[:3, 0], c2l[:3, 1], c2l[:3, 2] = right, down, fwd
        c2l[:3, 3] = radius * fwd + np.array([0., 0., height])
        m = K @ np.linalg.inv(c2l)
        l2i.append(m)
        i2l.append(np.linalg.inv(m))
    return np.stack(l2i), np.stack(i2l)


def analytic_sdf_volume(mapping, ground_z=-1.0, spheres=((6., 10., 0., 2.5), (-8., 4., -0.2, 1.5), (3., -12., 0.5, 2.0)),
                        boxes=((-4., 18., -1., 3., 2., 2.),), seed=0, noise=0.0):
    """SDF of ground plane + spheres + axis-aligned boxes sampled at the voxel lattice -> [H,W,Z] fp32."""
    H, W, Z = mapping.size_h, mapping.size_w, mapping.size_d
    g = torch.stack(torch.meshgrid(torch.arange(H, dtype=torch.float), torch.arange(W, dtype=torch.float),
                                   torch.arange(Z, dtype=torch.float), indexing='ij'), -1)
    p = mapping.grid2meter(g)
    sdf = p[..., 2] - ground_z
    for (sx, sy, sz, r) in spheres:
        sdf = torch.minimum(sdf, (p - torch.tensor([sx, sy, sz])).norm(dim=-1) - r)
    for (bx, by, bz, hx, hy, hz) in boxes:
        q = (p - torch.tensor([bx, by, bz])).abs() - torch.tensor([hx, hy, hz])
        sdf = torch.minimum(sdf, q.clamp(min=0).norm(dim=-1) + q.max(-1).values.clamp(max=0))
    if noise > 0:
        gen = torch.Generator().manual_seed(seed)
        sdf = sdf + noise * torch.randn(sdf.shape, generator=gen)
    return sdf.contiguous()


def pack_sdf_volume(sdf_hwz, zpitch):
    """[H,W,Z] -> the kernels' [H,W,zpitch] layout (pad zeroed)."""
    H, W, Z = sdf_hwz.shape
    out = torch.zeros(H, W, zpitch, dtype=sdf_hwz.dtype, device=sdf_hwz.device)
    out[..., :Z] = sdf_hwz
    return out


def pack_feat_volume(feat_chwz, feat_pitch):
    """[C,H,W,Z] -> channel-last [H,W,Z,feat_pitch] (pad zeroed)."""
    C, H, W, Z = feat_chwz.shape
    out = torch.zeros(H, W, Z, feat_pitch, dtype=feat_chwz.dtype, device=feat_chwz.device)
    out[..., :C] = feat_chwz.permute(1, 2, 3, 0)
    return out


def random_planes(mapping, C, scale=0.1, seed=0):
    gen = torch.Generator().manual_seed(seed)
    H, W, Z = mapping.size_h, mapping.size_w, mapping.size_d
    return [scale * torch.randn(n, C, generator=gen) for n in (H * W, Z * H, W * Z)]


def random_mlp(C, n_out, seed=0):
    gen = torch.Generator().manual_seed(seed + 1)
    lim = math.sqrt(6.0 / (C + C))
    w1 = (torch.rand(C, C, generator=gen) * 2 - 1) * lim
    b1 = 0.1 * torch.randn(C, generator=gen)
    w2 = (torch.rand(n_out, C, generator=gen) * 2 - 1) * math.sqrt(6.0 / (C + n_out))
    b2 = 0.1 * torch.randn(n_out, generator=gen)
    return w1, b1, w2, b2


def fpn_level_shapes(img_h, img_w, strides=(8, 16, 32, 64)):
    return [(math.ceil(img_h / s), math.ceil(img_w / s)) for s in strides]


def temporal_rig(yaws_deg=NUSC_YAWS, f=1266.0, cx=800.0, cy=450.0, height=1.5, radius=0.5, forward=0.5, yaw_deg=1.0):
    """img2prevImg / img2nextImg of camera_rig() under a small ego motion: the previous frame's ego pose is `forward`
    metres behind along the lidar y axis and yawed by -yaw_deg, the next one as far ahead and yawed by +yaw_deg.
    A pixel (u, v) at camera depth t maps to lidar2img @ inv(ego pose) @ img2lidar @ (u t, v t, t, 1).
    Returns (img2prevImg [N,4,4], img2nextImg [N,4,4]) float64 numpy."""
    l2i, i2l = camera_rig(yaws_deg, f, cx, cy, height, radius)
    out = []
    for sign in (-1.0, 1.0):
        a = np.deg2rad(sign * yaw_deg)
        pose = np.eye(4)
        pose[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        pose[1, 3] = sign * forward
        out.append(np.stack([l2i[c] @ np.linalg.inv(pose) @ i2l[c] for c in range(len(yaws_deg))]))
    return out[0], out[1]


def textured_images(n_img, H, W, seed=0, waves=6):
    """Smooth seeded RGB images [n_img, 3, H, W] fp32 in about [0.05, 0.95]: a sum of random plane waves with periods of
    tens to hundreds of pixels per channel, so bilinear colours and their differences vary smoothly and are not degenerate."""
    g = torch.Generator().manual_seed(seed)
    y = torch.arange(H, dtype=torch.float64)[:, None] / max(H, W)
    x = torch.arange(W, dtype=torch.float64)[None, :] / max(H, W)
    img = torch.full((n_img, 3, H, W), 0.5, dtype=torch.float64)
    for _ in range(waves):
        k = (torch.rand(n_img, 3, 2, generator=g, dtype=torch.float64) * 2 - 1) * 40.0      # radians across the image
        ph = torch.rand(n_img, 3, generator=g, dtype=torch.float64) * 6.283185307179586
        amp = 0.45 / waves * (0.5 + torch.rand(n_img, 3, generator=g, dtype=torch.float64))
        img += amp[..., None, None] * torch.sin(k[..., 0, None, None] * x + k[..., 1, None, None] * y + ph[..., None, None])
    return img.float().contiguous()
