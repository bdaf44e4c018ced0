"""Generate tests/golden/reference_golden_losses.npz and reference_multiloss_cfgs.json from the reference's loss terms.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_losses.py <path to the SelfOcc checkout>
loss/base_loss.py, rgb_loss_ms.py, edge_loss_3d_ms.py, eikonal_loss.py, second_grad_loss.py, sparsity_loss.py and
multi_loss.py are loaded by path as modules of a synthetic `loss` package and executed UNMODIFIED.  The stand-ins are those
of make_golden_reproj.py: an OPENOCC_LOSS whose register_module is the identity (plus a `build` by class name, which
MultiLoss calls), and a `utils.tb_wrapper.WrappedTBWriter` with an empty `_instance_dict` (no writer).  Inputs are seeded
and stored beside the outputs.
"""
import glob
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))
FILES = ('rgb_loss_ms', 'edge_loss_3d_ms', 'eikonal_loss', 'second_grad_loss', 'sparsity_loss', 'multi_loss')
# the small ray grid every golden case uses in place of the configs' img_size / ray_resize
IMG_SIZE, RAY_RESIZE, N_CLS = [48, 80], [6, 10], 5


def load_reference():
    classes = {}

    class _Reg:
        def register_module(self, *a, **k):
            return lambda cls: cls

        def build(self, cfg):
            cfg = dict(cfg)
            return classes[cfg.pop('type')](**cfg)
    lp = types.ModuleType('loss')
    lp.__path__ = []
    lp.OPENOCC_LOSS = _Reg()
    ut, tb = types.ModuleType('utils'), types.ModuleType('utils.tb_wrapper')
    ut.__path__ = []
    tb.WrappedTBWriter = type('WrappedTBWriter', (), {'_instance_dict': {}})
    sys.modules.update({'loss': lp, 'utils': ut, 'utils.tb_wrapper': tb})

    def load_as(rel, name):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod
    load_as('loss/base_loss.py', 'loss.base_loss')
    for f in FILES:
        m = load_as('loss/%s.py' % f, 'loss.' + f)
        classes.update({k: v for k, v in vars(m).items() if isinstance(v, type)})
    return classes


def make_inputs():
    """One seeded case: 2 cameras, a non-square 6x10 ray grid, 2 scales, 20x36 images under a 48x80 img_size."""
    g = torch.Generator().manual_seed(11)
    R = RAY_RESIZE[0] * RAY_RESIZE[1]
    ys, xs = torch.meshgrid(torch.arange(RAY_RESIZE[0]), torch.arange(RAY_RESIZE[1]), indexing='ij')
    rays_in = torch.stack([(xs.flatten() + 0.5) * IMG_SIZE[1] / RAY_RESIZE[1],
                           (ys.flatten() + 0.5) * IMG_SIZE[0] / RAY_RESIZE[0]], -1) + (torch.rand(R, 2, generator=g) - 0.5)
    rays_out = rays_in.clone()
    rays_out[::7, 0] -= 12.0                     # left of the image
    rays_out[3::7, 1] += 30.0                    # below the image
    rays_out[5, :] = torch.tensor([-0.5, IMG_SIZE[0] + 0.5])
    eik = torch.randn(40, 8, 3, generator=g) * 0.7
    eik[0, :3] = 0.                              # zero-norm rows
    eik[5, 2] = 0.
    sg = torch.randn(40, 8, 3, generator=g)
    sg[sg.abs() < 0.3] = 0.                      # exact zeros
    dens = torch.randn(6, 7, 5, generator=g)
    dens[dens.abs() < 0.3] = 0.
    colors = [torch.rand(1, 2, R, 3, generator=g) for _ in range(2)]
    gt = torch.rand(1, 2, 3, 20, 36, generator=g)
    curr = torch.rand(1, 2, 3, 20, 36, generator=g)
    depths = [0.5 + 20 * torch.rand(1, 2, R, generator=g) for _ in range(2)]
    accs = [torch.rand(1, 2, R, generator=g) for _ in range(2)]
    maxd = [20 + 10 * torch.rand(1, 2, R, generator=g) for _ in range(2)]
    sem_lab = torch.randint(0, N_CLS, (1, 2, IMG_SIZE[0], IMG_SIZE[1]), generator=g).to(torch.uint8)
    lab = sem_lab.long()[:, :, rays_in[:, 1].long(), rays_in[:, 0].long()]
    sem = torch.rand(1, 2, R, N_CLS, generator=g) * 1.3 - 0.15      # some outside [0, 1]
    onehot = torch.nn.functional.one_hot(lab, N_CLS).bool()
    # exactly at the clamp bounds where the gradient stays finite: 0 / 1 off / on the label class, 1e-6 on it
    sem[..., 0:4, :][~onehot[..., 0:4, :]] = 0.
    sem[..., 4:8, :][onehot[..., 4:8, :]] = 1.
    sem[..., 8:12, :][onehot[..., 8:12, :]] = float(np.float32(1e-6))
    return dict(rays_in=rays_in, rays_out=rays_out, eik=eik, sg=sg, dens=dens, colors=torch.stack(colors), gt=gt, curr=curr,
                depths=torch.stack(depths), accs=torch.stack(accs), maxd=torch.stack(maxd), sem_lab=sem_lab, sem=sem)


def golden():
    C = load_reference()
    inp = make_inputs()
    out = {k: v.numpy() for k, v in inp.items()}
    out.update(img_size=np.array(IMG_SIZE), ray_resize=np.array(RAY_RESIZE))
    leaf = lambda k: inp[k].clone().requires_grad_(True)

    def run(tag, loss, grads):
        loss.backward()
        out[tag + '_loss'] = np.array(float(loss.detach()))
        for name, t in grads.items():
            out['%s_grad_%s' % (tag, name)] = t.grad.numpy()

    for cls, key, name in (('EikonalLoss', 'eik_grad', 'eik'), ('SecondGradLoss', 'second_grad', 'sg'),
                           ('SoftSparsityLoss', 'density', 'dens')):
        x = leaf(name)
        run(cls, C[cls](weight=1.0)({key: x}), {name: x})
    metas = [dict(sem=inp['sem_lab'][0].numpy())]
    for rays in ('in', 'out'):
        for ssim in (0, 1):
            c = leaf('colors')
            m = C['RGBLossMS'](weight=1.0, img_size=IMG_SIZE, no_ssim=not ssim, ray_resize=RAY_RESIZE)
            run('RGBLossMS_ssim%d_rays%s' % (ssim, rays), m(dict(ms_colors=list(c.unbind(0)), ms_rays=inp['rays_' + rays],
                                                                 gt_imgs=inp['gt'])), {'colors': c})
        for inf in (0, 1):
            d, a, mx = leaf('depths'), leaf('accs'), leaf('maxd')
            keys = dict(curr_imgs='curr_imgs', ms_depths='ms_depths', ms_rays='ms_rays')
            if inf:
                keys.update(ms_accs='ms_accs', max_depths='max_depths')
            m = C['EdgeLoss3DMS'](weight=1.0, img_size=IMG_SIZE, ray_resize=RAY_RESIZE, use_inf_mask=bool(inf), input_dict=keys)
            run('EdgeLoss3DMS_inf%d_rays%s' % (inf, rays),
                m(dict(curr_imgs=inp['curr'], ms_depths=list(d.unbind(0)), ms_rays=inp['rays_' + rays], ms_accs=list(a.unbind(0)),
                       max_depths=list(mx.unbind(0)))), dict(depths=d, accs=a, maxd=mx) if inf else dict(depths=d))
    for cls in ('SemLossMS', 'SemCELossMS'):
        s = leaf('sem')
        run(cls, C[cls](weight=1.0, img_size=IMG_SIZE)(dict(sem=[s], metas=metas, ms_rays=inp['rays_in'])), {'sem': s})

    # every shipped config's loss dict; MultiLoss over its non-reprojection terms on the small case
    cfgs = {}
    for f in sorted(glob.glob(os.path.join(REF, 'config', '*', '*.py'))):
        if '_base_' in f:
            continue
        ns = {}
        exec(compile(open(f).read(), f, 'exec'), ns)
        if 'loss' in ns:
            cfgs[os.path.relpath(f, os.path.join(REF, 'config'))] = ns['loss']
    json.dump(cfgs, open(os.path.join(HERE, 'reference_multiloss_cfgs.json'), 'w'), indent=1, sort_keys=True)
    for name, loss_cfg in cfgs.items():
        tag = 'multi_' + os.path.splitext(os.path.basename(name))[0]
        terms = [small_cfg(c) for c in loss_cfg['loss_cfgs'] if not c['type'].startswith('ReprojLoss')]
        ml = C['MultiLoss'](terms)
        tot, d = ml(multi_inputs(inp))
        out[tag + '_total'] = np.array(float(tot))
        out[tag + '_names'] = np.array(list(d))
        out[tag + '_values'] = np.array(list(d.values()), dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, 'reference_golden_losses.npz'), **out)
    print('wrote loss golden:', len(out), 'arrays;', len(cfgs), 'configs')


def small_cfg(c):
    """A shipped term cfg on the golden case's grid: img_size / ray_resize replaced, everything else kept."""
    c = dict(c)
    for k, v in (('img_size', IMG_SIZE), ('ray_resize', RAY_RESIZE)):
        if k in c:
            c[k] = list(v)
    if c['type'] == 'EdgeLoss3DMS':
        c.setdefault('img_size', list(IMG_SIZE))
    return c


def multi_inputs(inp):
    """The head / dataset outputs the shipped terms read, under the configs' key names (the small case, one scale)."""
    return dict(eik_grad=inp['eik'], second_grad=inp['sg'], uniform_sdf=inp['dens'], ms_colors=[inp['colors'][0]],
                color_imgs=inp['gt'], curr_imgs=inp['curr'], ms_depths=[inp['depths'][0]], ms_rays=inp['rays_in'],
                sem=[inp['sem']], metas=[dict(sem=inp['sem_lab'][0].numpy())])


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'loss', 'multi_loss.py')):
        sys.exit('usage: python tests/golden/make_golden_losses.py <path to a huang-yh/SelfOcc checkout>')
    golden()
