"""fp64 restatement of the second-grad term (declared assumption, selfocc_b200/csrc/field_hess.cu): second_grad = the row
sums of the Hessian of the trilinear interpolant in metres, (Hxy + Hxz, Hxy + Hyz, Hxz + Hyz), zero padding outside the
volume, and SecondGradLoss's mean of |second_grad| with its gradient w.r.t. the sdf volume.

The points are given as grid coordinates (h, w, d) with the metre->grid slopes (kh, kw, kd) of each point, so the oracle
can run at exactly the sample points a kernel used (ops.render_train_probe)."""
import torch


def axis_slopes(grid, axes):
    """[N, 3] metre->grid slopes of grid points [N, 3] (h, w, d) under axes = three (offset, size0, k0, k1) of the volume's
    axis maps: k1 in the outer ring (|g - offset| > size0, k1 > 0), k0 inside."""
    out = []
    for i, (offset, size0, k0, k1) in enumerate(axes):
        ring = (grid[:, i] - offset).abs() > size0
        out.append(torch.where(ring & (k1 > 0), torch.full_like(grid[:, i], k1), torch.full_like(grid[:, i], k0)))
    return torch.stack(out, -1)


def second_grad_ref(vol, grid, slopes, absolute=False):
    """vol [H, W, Z] fp64, grid / slopes [N, 3] -> [N, 3] second_grad in fp64.  absolute: the same sums with every corner
    term replaced by its magnitude (|coefficient| |value|), the scale of a component's rounding error."""
    H, W, Z = vol.shape
    g = grid.double()
    fl = torch.floor(g)
    f = g - fl
    i0 = fl.long()
    s_hw = s_hz = s_wz = 0.
    for i in (0, 1):
        for j in (0, 1):
            for k in (0, 1):
                h, w, z = i0[:, 0] + i, i0[:, 1] + j, i0[:, 2] + k
                inside = (h >= 0) & (h < H) & (w >= 0) & (w < W) & (z >= 0) & (z < Z)
                a = vol[h.clamp(0, H - 1), w.clamp(0, W - 1), z.clamp(0, Z - 1)] * inside
                si, sj, sk = (1. if i else -1.), (1. if j else -1.), (1. if k else -1.)
                wh, ww, wz = (f[:, 0] if i else 1 - f[:, 0]), (f[:, 1] if j else 1 - f[:, 1]), (f[:, 2] if k else 1 - f[:, 2])
                c_hw, c_hz, c_wz = si * sj * wz, si * sk * ww, sj * sk * wh
                if absolute:
                    a, c_hw, c_hz, c_wz = a.abs(), c_hw.abs(), c_hz.abs(), c_wz.abs()
                s_hw = s_hw + c_hw * a
                s_hz = s_hz + c_hz * a
                s_wz = s_wz + c_wz * a
    sl = slopes.double().abs() if absolute else slopes.double()
    kh, kw, kd = sl[:, 0], sl[:, 1], sl[:, 2]
    Hxy, Hxz, Hyz = kw * kh * s_hw, kw * kd * s_wz, kh * kd * s_hz
    return torch.stack([Hxy + Hxz, Hxy + Hyz, Hxz + Hyz], -1)


def second_grad_mean_ref(vol, grid, slopes, g_mean=1.0, amb_rtol=1e-5, chunk=1 << 20):
    """SecondGradLoss on the points: (mean of |second_grad| over N x 3 elements, d (g_mean * mean) / d vol, bound, n_amb).

    An element whose fp64 value lies within amb_rtol of its magnitude form (second_grad_ref(absolute=True)) has no sign a
    fp32 evaluation can be held to: the gradient takes its fp64 sign (0 at 0), and what a fp32 evaluation with the other
    sign would change on each voxel, 2 g_mean / (3 N) times its corner coefficients' magnitudes, is summed in `bound`
    [H, W, Z] (n_amb such elements)."""
    n = grid.shape[0]
    count = 3 * n
    tot = torch.zeros((), dtype=torch.float64, device=vol.device)
    grad = torch.zeros_like(vol, dtype=torch.float64)
    bound = torch.zeros_like(vol, dtype=torch.float64)
    n_amb = 0
    scale = g_mean / count
    for b in range(0, n, chunk):
        gr, sl = grid[b:b + chunk], slopes[b:b + chunk]
        v = vol.detach().double().requires_grad_(True)
        x = second_grad_ref(v, gr, sl)
        with torch.no_grad():
            mag = second_grad_ref(v.detach(), gr, sl, absolute=True)
            amb = x.detach().abs() <= amb_rtol * mag
        tot += x.detach().abs().sum()
        n_amb += int(amb.sum())
        grad += torch.autograd.grad((x * torch.sign(x.detach())).sum() * scale, v)[0]
        if amb.any():
            # |d x_e / d vol| summed over the ambiguous elements: the coefficient magnitudes times a unit volume
            u = torch.ones_like(vol, dtype=torch.float64).requires_grad_(True)
            xa = second_grad_ref(u, gr, sl, absolute=True)
            bound += torch.autograd.grad((xa * amb).sum() * 2 * abs(scale), u)[0]
    return tot / count, grad, bound, n_amb
