"""Generate tests/golden/reference_golden_reproj.npz and reference_loss_cfgs.json from the reference's reprojection losses.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_reproj.py <path to the SelfOcc checkout>
The loss modules are loaded by file path and executed unmodified; inputs are seeded and stored beside the outputs.
"""
import importlib.util
import os
import sys
import numpy as np
import torch

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))


def reproj_golden():
    """Pins oracle/reproj.py to the reference's two reprojection losses, executed UNMODIFIED:
    loss/reproj_loss_mono_multi_new_combine.py and loss/reproj_loss_mono_multi_new.py with loss/base_loss.py, loaded by
    path as modules of a synthetic `loss` package whose OPENOCC_LOSS is a stand-in with an identity register_module, and
    with `utils.tb_wrapper.WrappedTBWriter` a stand-in with an empty `_instance_dict` (no writer).  One seeded small case
    (2 cameras, a 6x10 ray grid, S = 16, textured 20x36 images under a 48x80 img_size) whose reprojections leave the image,
    fall behind the camera and leave some rays without a valid sample; both variants x no_ssim x no_automask x deltas.
    Writes tests/golden/reference_golden_reproj.npz (inputs, loss, d loss / d weights) and reference_loss_cfgs.json (the
    reprojection loss dicts of the shipped configs)."""
    import glob
    import json
    import types
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from selfocc_b200 import synth

    class _Reg:
        def register_module(self, *a, **k):
            return lambda cls: cls
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
    comb = load_as('loss/reproj_loss_mono_multi_new_combine.py', 'loss.reproj_loss_mono_multi_new_combine')
    mnew = load_as('loss/reproj_loss_mono_multi_new.py', 'loss.reproj_loss_mono_multi_new')

    g = torch.Generator().manual_seed(5)
    N, ray_resize, S, img_size, HW = 2, [6, 10], 16, [48, 80], (20, 36)
    R = ray_resize[0] * ray_resize[1]
    ys, xs = torch.meshgrid(torch.arange(ray_resize[0]), torch.arange(ray_resize[1]), indexing='ij')
    ms_rays = torch.stack([(xs.flatten() + 0.5) * img_size[1] / ray_resize[1], (ys.flatten() + 0.5) * img_size[0] / ray_resize[0]],
                          -1).float() + 0.3 * torch.rand(R, 2, generator=g)
    # camera 0: a physical rig under ego motion; camera 1: large pixel shifts so that rays at the right / bottom have no
    # valid sample in either frame, and a 0.5 m depth offset that puts near samples behind the camera
    p0, n0 = synth.temporal_rig(yaws_deg=(0.,), f=40.0, cx=40.0, cy=24.0, forward=0.5, yaw_deg=3.0)
    p1, n1 = np.eye(4), np.eye(4)
    p1[0, 2], p1[2, 3] = 35.0, -0.5
    n1[1, 2], n1[2, 3] = 20.0, 0.5
    img2prev, img2next = np.concatenate([p0, p1[None]]), np.concatenate([n0, n1[None]])
    metas = [dict(img2prevImg=list(img2prev), img2nextImg=list(img2next))]
    imgs = [synth.textured_images(N, *HW, seed=s)[None] for s in (1, 2, 3)]
    ts = (0.05 + 30.0 * torch.rand(N, R * S, generator=g) ** 2)
    ts[:, :S] = 0.2                                         # a ray whose samples all sit at 0.2 m
    weights = torch.rand(N, R * S, generator=g) * (torch.rand(N, R * S, generator=g) < 0.7)
    weights[:, S:2 * S] = 0.                                # a ray whose weights are all zero
    deltas = 0.05 + torch.rand(N, R * S, generator=g)
    deltas[:, ::7] = 0.                                     # delta < eps: the sample is dropped
    ray_idx = torch.arange(R).repeat_interleave(S)
    out = dict(ms_rays=ms_rays.numpy(), img2prev=img2prev, img2next=img2next, curr=imgs[0].numpy(), prev=imgs[1].numpy(),
               next=imgs[2].numpy(), ts=ts.numpy(), weights=weights.numpy(), deltas=deltas.numpy(),
               img_size=np.array(img_size), ray_resize=np.array(ray_resize))
    for variant, mod, cls in (('combine', comb, 'ReprojLossMonoMultiNewCombine'), ('multi_new', mnew, 'ReprojLossMonoMultiNew')):
        for no_ssim in (False, True):
            for no_automask in (False, True):
                for use_deltas in (False, True):
                    keys = {k: k for k in ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')}
                    if use_deltas:
                        keys['deltas'] = 'deltas'
                    loss_mod = getattr(mod, cls)(weight=1.0, input_dict=keys, no_ssim=no_ssim, img_size=img_size,
                                                 ray_resize=ray_resize, no_automask=no_automask)
                    w = weights.clone().requires_grad_(True)
                    inputs = dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], ray_indices=[ray_idx] * N,
                                  weights=list(w.unbind(0)), ts=list(ts.unbind(0)), metas=metas, ms_rays=ms_rays,
                                  deltas=list(deltas.unbind(0)))
                    loss = loss_mod(inputs)
                    loss.backward()
                    tag = '%s_ssim%d_auto%d_deltas%d' % (variant, not no_ssim, not no_automask, use_deltas)
                    out[tag + '_loss'] = np.array(float(loss))
                    out[tag + '_grad'] = w.grad.numpy()
    np.savez_compressed(os.path.join(HERE, 'reference_golden_reproj.npz'), **out)
    cfgs = {}
    for f in sorted(glob.glob(os.path.join(REF, 'config', '*', '*.py'))):
        if '_base_' in f:
            continue
        ns = {}
        exec(compile(open(f).read(), f, 'exec'), ns)
        for l in ns.get('loss', {}).get('loss_cfgs', []):
            if l['type'].startswith('ReprojLoss'):
                cfgs[os.path.relpath(f, os.path.join(REF, 'config'))] = l
    json.dump(cfgs, open(os.path.join(HERE, 'reference_loss_cfgs.json'), 'w'), indent=1, sort_keys=True)
    print('wrote reproj golden:', len(out), 'arrays;', len(cfgs), 'loss configs')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'loss', 'reproj_loss_mono_multi_new_combine.py')):
        sys.exit('usage: python tests/golden/make_golden_reproj.py <path to a huang-yh/SelfOcc checkout>')
    reproj_golden()
