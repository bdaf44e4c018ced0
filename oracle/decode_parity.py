"""Oracle-side helpers for the TPV decode gate (test infrastructure, see oracle/__init__.py).

``render.tpv_decode_ref`` restated one slab of h rows at a time, so that the fp64 decode of a shipped volume
(257 x 257 x 31 voxels x 96 channels) and its autograd need tens of MB per activation instead of the whole
[H, W, Z, C] broadcast sum.  Everything runs in the dtype and on the device of its inputs: the tests pass fp64 tensors on
the GPU.  Outputs are channel-last, [H, W, Z, 1 + n_feat], the layout the decoded volume is compared in.
"""
import torch
import torch.nn.functional as F

PLANE_NAMES = ('tpv_hw', 'tpv_zh', 'tpv_wz')
GRAD_NAMES = PLANE_NAMES + ('w1', 'b1', 'w2', 'b2')
# first-layer pre-activation intervals the activation's error is reported on (softplus and sigmoid lose relative accuracy
# towards the negative end when they are formed through 1 + exp(x) in fp32)
BUCKETS = ((-float('inf'), -16.0), (-16.0, -12.0), (-12.0, -8.0), (-8.0, -4.0), (-4.0, 0.0), (0.0, 20.0), (20.0, float('inf')))


def preactivation(tpv_hw, tpv_zh, tpv_wz, sizes, h0, h1):
    """f[h0:h1] = hw[h, w] + zh[z, h] + wz[w, z]  ->  [h1 - h0, W, Z, C]."""
    H, W, Z = sizes
    C = tpv_hw.shape[-1]
    return (tpv_hw.reshape(H, W, 1, C)[h0:h1] + tpv_zh.reshape(Z, H, 1, C).permute(1, 2, 0, 3)[h0:h1]
            + tpv_wz.reshape(1, W, Z, C))


def _mlp(f, w1, b1, w2, b2):
    return F.linear(F.softplus(F.linear(F.softplus(f), w1, b1)), w2, b2)


def decode_slabwise(tpv_hw, tpv_zh, tpv_wz, sizes, w1, b1, w2, b2, slab=8):
    """Decoded volume [H, W, Z, 1 + n_feat]."""
    H = sizes[0]
    with torch.no_grad():
        return torch.cat([_mlp(preactivation(tpv_hw, tpv_zh, tpv_wz, sizes, h0, min(H, h0 + slab)), w1, b1, w2, b2)
                          for h0 in range(0, H, slab)], 0)


def decode_grads_slabwise(tpv_hw, tpv_zh, tpv_wz, sizes, w1, b1, w2, b2, g_out, slab=8):
    """Gradients of <decode, g_out> (g_out [H, W, Z, 1 + n_feat]) w.r.t. the three planes and the four MLP tensors, in the
    order of GRAD_NAMES, and b1_mass [C].  The loss is a sum over voxels, so the gradient is the sum of the slabs' gradients.
    d/d b1[j] is the plain sum over voxels of the hidden pre-activation's gradient: signed terms that cancel, so the entry
    itself is no stable scale for its error; b1_mass[j] is the sum of the terms' magnitudes."""
    H = sizes[0]
    ins = [t.detach().requires_grad_(True) for t in (tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2)]
    grads = [torch.zeros_like(t) for t in ins]
    b1_mass = torch.zeros_like(b1)
    for h0 in range(0, H, slab):
        h1 = min(H, h0 + slab)
        z1 = F.linear(F.softplus(preactivation(*ins[:3], sizes, h0, h1)), ins[3], ins[4])
        out = F.linear(F.softplus(z1), ins[5], ins[6])
        *gs, g_z1 = torch.autograd.grad((out * g_out[h0:h1]).sum(), ins + [z1])
        for acc, g in zip(grads, gs):
            acc += g
        b1_mass += g_z1.abs().sum((0, 1, 2))
    return grads, b1_mass


def bucket_errors(got, ref, pre):
    """Per BUCKETS interval of ``pre``: (elements, max |got - ref|, max |got - ref| / |ref|); ``ref`` must be nonzero."""
    got, rows = got.to(ref), []
    err = (got - ref).abs()
    for lo, hi in BUCKETS:
        sel = (pre >= lo) & (pre < hi)
        n = int(sel.sum())
        rows.append((n, float(err[sel].max()) if n else 0.0, float((err[sel] / ref[sel].abs()).max()) if n else 0.0))
    return rows


def slice_errors(got, ref, dim):
    """Error of every slice of ``ref`` along ``dim`` relative to that slice's own max-abs: max_i |got - ref| / max_i |ref|
    per index of ``dim``.  Slices whose reference is exactly zero are returned as 0 (nothing to be relative to)."""
    got = got.to(ref)
    other = [d for d in range(ref.dim()) if d != dim]
    scale = ref.abs().amax(other) if other else ref.abs()
    err = (got - ref).abs().amax(other) if other else (got - ref).abs()
    return torch.where(scale > 0, err / scale.clamp_min(torch.finfo(ref.dtype).tiny), torch.zeros_like(err))
