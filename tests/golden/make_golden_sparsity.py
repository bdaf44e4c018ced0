"""Generate tests/golden/reference_golden_sparsity.npz from the reference's SparsityLoss, HardSparsityLoss and
AdaptiveSparsityLoss (loss/sparsity_loss.py).

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_sparsity.py <path to the SelfOcc checkout>
The loss files are loaded UNMODIFIED with make_golden_losses.py's stand-ins.  Inputs are seeded and stored beside the
outputs.  Cases:
  * SparsityLoss at scale 0.1 and 1.0 on a lattice with entries past the fp32 cosh range (|x| / (2 scale) > 89): there the
    reference's value is 0 and its gradient NaN (cosh backward: 0 * sinh = 0 * inf);
  * HardSparsityLoss without a crop, with a crop on every border, with a crop that covers the whole lattice, with the relu
    inactive, and at a small slope; the reference writes the crop into its input, so each call gets a copy;
  * AdaptiveSparsityLoss with a few masked samples per ray (some rays with none), and with an empty mask (NaN value).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_losses import REF, load_reference  # noqa: E402

LATTICE = (6, 7, 5)
HARD_CASES = {                                       # tag -> (scale, thresh, crop)
    'nocrop': (1.0, 0.2, [[0, 0], [0, 0], [0, 0]]),
    'crop': (1.0, 0.05, [[1, 2], [2, 1], [1, 1]]),
    'allcrop': (0.02, 0.1, [[3, 3], [0, 0], [0, 0]]),
    'inactive': (1.0, 0.9, [[1, 0], [0, 0], [0, 2]]),
    'slope': (0.05, 0.2, [[0, 1], [0, 0], [2, 0]]),
}
SPARSITY_SCALES = {'s01': 0.1, 's1': 1.0}
N_CAM, R, S, SLACK = 2, 12, 16, 4.0


def make_inputs():
    g = torch.Generator().manual_seed(23)
    dens = torch.randn(*LATTICE, generator=g) * 2.0
    dens[dens.abs() < 0.2] = 0.
    dens.view(-1)[0:132:11] = torch.tensor([20., -25., 60., -1e3, 1e4, 18.5, -17.0, 3e38, -200., 40., 90., -90.])
    ts = (0.5 + 40 * torch.rand(N_CAM, R, S, generator=g)).sort(-1).values
    depths = 1 + 30 * torch.rand(1, N_CAM, R, generator=g)
    depths[0, 0, :3] = 100.                           # rays with no masked sample
    sdfs = torch.randn(N_CAM, R, S, generator=g)
    sdfs[sdfs.abs() < 0.1] = 0.
    return dict(dens=dens, ts=ts.reshape(N_CAM, R * S), depths=depths, sdfs=sdfs.reshape(N_CAM, R * S),
                depths_far=torch.full((1, N_CAM, R), 100.))


def golden():
    C = load_reference()
    inp = make_inputs()
    out = {k: v.numpy() for k, v in inp.items()}
    out['slack'] = np.array(SLACK)

    def run(tag, loss, grads):
        loss.backward()
        out[tag + '_loss'] = np.array(float(loss.detach()))
        for name, t in grads.items():
            out['%s_grad_%s' % (tag, name)] = t.grad.numpy()

    for tag, scale in SPARSITY_SCALES.items():
        x = inp['dens'].clone().requires_grad_(True)
        run('SparsityLoss_' + tag, C['SparsityLoss'](weight=1.0, scale=scale)({'density': x}), {'dens': x})
    for tag, (scale, thresh, crop) in HARD_CASES.items():
        x = inp['dens'].clone().requires_grad_(True)
        out['HardSparsityLoss_%s_cfg' % tag] = np.array([scale, thresh] + [c for row in crop for c in row], dtype=np.float64)
        m = C['HardSparsityLoss'](weight=1.0, scale=scale, thresh=thresh, crop=crop)
        run('HardSparsityLoss_' + tag, m({'density': x.clone()}), {'dens': x})      # the reference crops its input in place
    for tag, dk in (('masked', 'depths'), ('empty', 'depths_far')):
        s = inp['sdfs'].clone().requires_grad_(True)
        m = C['AdaptiveSparsityLoss'](weight=1.0, slack=SLACK)
        run('AdaptiveSparsityLoss_' + tag, m(dict(sdfs=list(s.unbind(0)), ts=list(inp['ts'].unbind(0)), ms_depths=[inp[dk]])),
            {'sdfs': s})
    np.savez_compressed(os.path.join(HERE, 'reference_golden_sparsity.npz'), **out)
    print('wrote sparsity golden:', len(out), 'arrays')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'loss', 'sparsity_loss.py')):
        sys.exit('usage: python tests/golden/make_golden_sparsity.py <path to a huang-yh/SelfOcc checkout>')
    golden()
