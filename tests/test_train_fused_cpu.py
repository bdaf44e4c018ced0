"""The fused training objective off the GPU: the argument checks of so_render_train_objective_forward / _backward (every
case fails or returns before any launch: the ray count is 0), and which objectives fuse_objective accepts."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest

from test_render_args_cpu import ONE, _desc, _params, _rays

HERE = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
INVALID, UNSUPPORTED = -1, -2


def _objective(**kw):
    from selfocc_b200 import _lib
    ob = _lib.ObjectiveDesc()
    ob.reproj_mode, ob.eikonal = 0, 1
    ob.pix = ob.img2prev = ob.img2next = ob.curr_imgs = ob.prev_imgs = ob.next_imgs = 16
    ob.img_h, ob.img_w, ob.size_h, ob.size_w = 96, 200, 768.0, 1600.0
    ob.workspace, ob.workspace_bytes = 16, 0
    for k, v in kw.items():
        setattr(ob, k, v)
    return ob


def _fwd(lib, ob=None, rd=None, pr=None, stats=ONE, colours=None, mean=ONE):
    ob = _objective() if ob is None else ob
    rd, pr = _rays(**(rd or {})), _params(**(pr or {}))
    n = None
    return lib.so_render_train_objective_forward(ONE, n, C.byref(_desc()), ONE, n, C.byref(rd), C.byref(pr), n, n,
                                                 None if ob == 'null' else C.byref(ob), n, n, n, n, n, n, n, n, n, n, n,
                                                 stats, colours, mean, ONE, n, n)


def _bwd(lib, ob=None, rd=None, pr=None, stats=ONE, g_stats=ONE, g_mean=ONE, g_inv_s=None):
    ob = _objective() if ob is None else ob
    rd, pr = _rays(**(rd or {})), _params(**(pr or {}))
    n = None
    return lib.so_render_train_objective_backward(ONE, n, C.byref(_desc()), ONE, n, C.byref(rd), C.byref(pr), n, n,
                                                  None if ob == 'null' else C.byref(ob), n, n, n, n, stats, g_stats, g_mean,
                                                  ONE, n, g_inv_s, ONE, n)


@pytest.fixture(scope='module')
def lib():
    from selfocc_b200 import _lib
    return _lib.load()


def test_valid_calls_without_rays_return_ok(lib):
    assert _fwd(lib) == 0
    assert _bwd(lib) == 0
    assert _bwd(lib, g_inv_s=ONE) == 0
    assert _fwd(lib, _objective(reproj_mode=-1), stats=None) == 0         # eikonal only
    assert _bwd(lib, _objective(reproj_mode=-1, eikonal=0), stats=None, g_stats=None, g_mean=None) == 0
    assert _fwd(lib, _objective(reproj_mode=1, eikonal=0), mean=None) == 0


@pytest.mark.parametrize('case, code', [
    (dict(ob='null'), INVALID),
    (dict(ob=dict(reproj_mode=2)), INVALID),
    (dict(ob=dict(eikonal=2)), INVALID),
    (dict(ob=dict(pix=0)), INVALID),
    (dict(ob=dict(img2next=0)), INVALID),
    (dict(ob=dict(prev_imgs=0)), INVALID),
    (dict(ob=dict(curr_imgs=18)), INVALID),                     # misaligned float operand
    (dict(ob=dict(img_h=0)), INVALID),
    (dict(ob=dict(size_w=0.0)), INVALID),
    (dict(ob=dict(size_h=float('inf'))), INVALID),
    (dict(ob=dict(img_h=50000, img_w=50000)), UNSUPPORTED),
    (dict(stats=None), INVALID),
    (dict(mean=None), INVALID),
    (dict(ob=dict(workspace=0)), INVALID),
    (dict(ob=dict(workspace=20)), INVALID),                     # not 8-byte aligned
    (dict(ob=dict(workspace_bytes=8 * 3), rd=dict(ray_count=4)), INVALID),
    (dict(pr=dict(num_samples=512)), UNSUPPORTED),              # S <= 256, the training render's bound
    (dict(pr=dict(num_samples=0)), INVALID),
    (dict(rd=dict(ray_count=5)), INVALID),                      # beyond n_cam * rays_per_cam
])
def test_forward_refuses_bad_arguments(lib, case, code):
    case = dict(case)
    if 'ob' in case and case['ob'] != 'null':
        case['ob'] = _objective(**case['ob'])
    assert _fwd(lib, **case) == code


@pytest.mark.parametrize('case, code', [
    (dict(ob='null'), INVALID),
    (dict(ob=dict(reproj_mode=-2)), INVALID),
    (dict(ob=dict(next_imgs=0)), INVALID),
    (dict(ob=dict(img_w=-1)), INVALID),
    (dict(stats=None), INVALID),
    (dict(g_stats=None), INVALID),
    (dict(g_mean=C.c_void_p(18)), INVALID),
    (dict(g_inv_s=ONE, ob=dict(workspace=0)), INVALID),         # the per-ray inv_s values need the workspace
    (dict(g_inv_s=ONE, ob=dict(workspace_bytes=8 * 3), rd=dict(ray_count=4)), INVALID),
    (dict(pr=dict(num_samples=300)), UNSUPPORTED),
])
def test_backward_refuses_bad_arguments(lib, case, code):
    case = dict(case)
    if 'ob' in case and case['ob'] != 'null':
        case['ob'] = _objective(**case['ob'])
    assert _bwd(lib, **case) == code


# ------------------------------------------------------------------------------------------------ fuse_objective
def _head(two_split=False, sample_sdf=False):
    return SimpleNamespace(two_split=two_split, img2lidar=SimpleNamespace(two_split=True), return_sample_sdf=sample_sdf,
                           fused_objective=None)


def _multiloss(cfgs):
    from selfocc_b200.loss import MultiLoss
    return MultiLoss(cfgs)


@pytest.mark.parametrize('name', sorted(CFGS))
def test_every_shipped_objective_can_be_fused(name):
    from selfocc_b200.loss import fuse_objective
    cfgs = CFGS[name]['loss_cfgs']
    head = _head()
    rec = fuse_objective(head, _multiloss(cfgs))
    reproj = next(c for c in cfgs if c['type'].startswith('ReprojLoss'))
    assert head.fused_objective is rec
    assert rec == dict(mode='combine' if reproj['type'] == 'ReprojLossMonoMultiNewCombine' else 'multi_new',
                       img_size=tuple(reproj['img_size']), eikonal=any(c['type'] == 'EikonalLoss' for c in cfgs))


R_COMBINE = dict(type='ReprojLossMonoMultiNewCombine', img_size=[768, 1600], ray_resize=[48, 100])
R_MULTI = dict(type='ReprojLossMonoMultiNew', img_size=[768, 1600], ray_resize=[48, 100])
EIK = dict(type='EikonalLoss', weight=0.1)
DEFAULT_IN = {k: k for k in ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')}


@pytest.mark.parametrize('cfgs, head', [
    ([R_COMBINE, R_MULTI, EIK], {}),                                                        # two reprojection terms
    ([R_COMBINE, EIK, EIK], {}),                                                            # two eikonal terms
    ([dict(R_COMBINE, input_dict=dict(DEFAULT_IN, deltas='deltas')), EIK], {}),            # deltas input
    ([dict(R_MULTI, input_dict=dict(DEFAULT_IN, weights='other_weights')), EIK], {}),      # weights from elsewhere
    ([R_COMBINE, dict(EIK, input_dict={'eik_grad': 'second_grad'})], {}),                   # eikonal of another tensor
    ([R_COMBINE, EIK, dict(type='SecondGradLoss', input_dict={'second_grad': 'eik_grad'})], {}),   # another per-sample reader
    ([R_COMBINE, EIK], dict(two_split=True)),
    ([R_COMBINE, EIK], dict(sample_sdf=True)),
])
def test_fuse_objective_refuses_unsupported_objectives(cfgs, head):
    from selfocc_b200.loss import fuse_objective
    h = _head(**head)
    with pytest.raises(NotImplementedError):
        fuse_objective(h, _multiloss(cfgs))
    assert h.fused_objective is None


def test_objective_without_per_sample_terms_fuses_to_nothing():
    from selfocc_b200.loss import fuse_objective
    assert fuse_objective(_head(), _multiloss([dict(type='SecondGradLoss')])) == dict(mode=None, img_size=None, eikonal=False)
