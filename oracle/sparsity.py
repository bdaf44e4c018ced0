"""Oracle: the sparsity terms of loss/sparsity_loss.py (test infrastructure; any dtype, any device; fp64 for the reference
values), with autograd through the density / sdf input:
  * sparsity_ref          loss/sparsity_loss.py:24-27     mean sech^2(x / (2 scale)), in a form that stays finite
  * hard_sparsity_ref     loss/sparsity_loss.py:46-63     relu(mean sigmoid(-scale x') - thresh), x' = x with the crop
                                                          borders set to 100 (on a copy: the input is not written)
  * adaptive_sparsity_ref loss/sparsity_loss.py:102-114   mean relu(-sdf) over the samples with ts > depth + slack
Pinned to the reference by tests/golden/reference_golden_sparsity.npz (tests/golden/make_golden_sparsity.py).
"""
import torch


def sparsity_ref(x, scale):
    """1 / cosh(u)^2, u = x / (2 scale), as 4 e / (1 + e)^2 with e = exp(-2|u|): the reference's value wherever its cosh is
    finite, and 0 (with a 0 gradient) where cosh overflows and the reference gives 1 / inf = 0."""
    e = torch.exp(-2 * (x / (2.0 * scale)).abs())
    return (4 * e / (1 + e) ** 2).mean()


def hard_sparsity_ref(x, scale=1.0, thresh=0.2, crop=((0, 0), (0, 0), (0, 0))):
    """x [H, W, D]; crop [[h0, h1], [w0, w1], [d0, d1]], a border is cropped where its value is > 0."""
    m = torch.ones_like(x, dtype=torch.bool)
    (h0, h1), (w0, w1), (d0, d1) = crop
    if h0 > 0:
        m[:h0] = False
    if h1 > 0:
        m[-h1:] = False
    if w0 > 0:
        m[:, :w0] = False
    if w1 > 0:
        m[:, -w1:] = False
    if d0 > 0:
        m[..., :d0] = False
    if d1 > 0:
        m[..., -d1:] = False
    xc = torch.where(m, x, torch.full_like(x, 100.0))          # out of place: no gradient reaches the cropped cells
    return torch.relu(torch.sigmoid(-scale * xc).mean() - thresh)


def adaptive_sparsity_ref(sdfs, ts, depths, slack=4.0):
    """sdfs, ts: per camera R * S samples ray-major; depths [1, N, R].  NaN when no sample is behind depth + slack."""
    bs, n, R = depths.shape
    t = torch.stack(list(ts)).reshape(bs, n, R, -1)
    s = torch.stack(list(sdfs)).reshape(bs, n, R, -1)
    mask = t > (depths + slack).unsqueeze(-1)
    return torch.relu(-s[mask]).mean()
