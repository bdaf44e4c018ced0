"""SecondGradLoss fused into the training render, off the GPU: fuse_objective's second_grad keyword and its refusals, the
second-grad fields of so_objective_desc and their argument checks (every case fails or returns before any launch: the ray
count is 0), and the fp64 restatement in oracle/second_grad.py."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest
import torch

from test_render_args_cpu import ONE
from test_train_fused_cpu import _bwd, _fwd, _objective

HERE = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
INVALID = -1
SG = dict(type='SecondGradLoss', weight=0.01)
EIK = dict(type='EikonalLoss', weight=0.1)
R_COMBINE = dict(type='ReprojLossMonoMultiNewCombine', img_size=[768, 1600], ray_resize=[48, 100])


@pytest.fixture(scope='module')
def lib():
    from selfocc_b200 import _lib
    return _lib.load()


# ------------------------------------------------------------------------------------------------ fuse_objective
def _head(second_grad=True, assumption=True):
    return SimpleNamespace(two_split=False, img2lidar=SimpleNamespace(two_split=True), return_sample_sdf=False,
                           return_second_grad=second_grad, second_grad_assumption=assumption, fused_objective=None)


def _multiloss(cfgs):
    from selfocc_b200.loss import MultiLoss
    return MultiLoss(cfgs)


SG_CFGS = sorted(n for n in CFGS if any(c['type'] == 'SecondGradLoss' for c in CFGS[n]['loss_cfgs']))


def test_the_shipped_second_grad_objectives_are_the_five_configs():
    assert [n.split('/')[-1] for n in SG_CFGS] == ['kitti_novel_depth.py', 'kitti_occ.py', 'nuscenes_novel_depth.py',
                                                   'nuscenes_occ.py', 'nuscenes_occ_bev.py']


@pytest.mark.parametrize('name', SG_CFGS)
def test_without_the_keyword_the_record_is_unchanged(name):
    from selfocc_b200.loss import fuse_objective
    cfgs = CFGS[name]['loss_cfgs']
    rec = fuse_objective(_head(), _multiloss(cfgs))
    assert set(rec) == {'mode', 'img_size', 'eikonal'}
    assert fuse_objective(_head(), _multiloss([SG])) == dict(mode=None, img_size=None, eikonal=False)


@pytest.mark.parametrize('name', SG_CFGS)
def test_every_shipped_second_grad_objective_fuses_its_second_grad_term(name):
    from selfocc_b200.loss import fuse_objective
    cfgs = CFGS[name]['loss_cfgs']
    head = _head()
    plain = fuse_objective(_head(), _multiloss(cfgs))
    rec = fuse_objective(head, _multiloss(cfgs), second_grad=True)
    assert head.fused_objective is rec
    assert rec == dict(plain, second_grad=True)


def test_the_keyword_without_a_second_grad_term_records_it_off():
    from selfocc_b200.loss import fuse_objective
    rec = fuse_objective(_head(second_grad=False, assumption=False), _multiloss([R_COMBINE, EIK]), second_grad=True)
    assert rec == dict(mode='combine', img_size=(768, 1600), eikonal=True, second_grad=False)


@pytest.mark.parametrize('cfgs, head', [
    ([R_COMBINE, EIK, dict(SG, input_dict={'second_grad': 'eik_grad'})], {}),        # another tensor
    ([R_COMBINE, EIK, dict(SG, input_dict={'second_grad': 'other'})], {}),
    ([R_COMBINE, EIK, SG, SG], {}),                                                   # two second-grad terms
    ([R_COMBINE, EIK, SG], dict(second_grad=False)),                                  # head without return_second_grad
    ([R_COMBINE, EIK, SG], dict(assumption=False)),                                   # head without the opt-in
])
def test_the_keyword_refuses_unsupported_second_grad_terms(cfgs, head):
    from selfocc_b200.loss import fuse_objective
    h = _head(**head)
    with pytest.raises(NotImplementedError):
        fuse_objective(h, _multiloss(cfgs), second_grad=True)
    assert h.fused_objective is None


def test_second_grad_loss_reads_the_fused_mean():
    from selfocc_b200.loss import SecondGradLoss
    term = SecondGradLoss(weight=0.25)
    m = torch.tensor(0.5, dtype=torch.float32)
    assert term({'second_grad_mean': m}).item() == 0.125
    inputs = {'second_grad_mean': m, 'ray_indices': [torch.zeros(12, dtype=torch.long)] * 2}
    (pay, full), = term.local_payload(inputs, (0, 3, 4))
    assert full == 3 and pay.shape == (1, 1, 2)
    assert pay.flatten().tolist() == [0.5 * 72, 72.0]                # mean x this rank's 2 x 12 x 3 elements, and the count
    assert term.from_gathered([pay.expand(3, 1, 2)], inputs).item() == 0.125


# ------------------------------------------------------------------------------------------------ C ABI
def test_the_second_grad_fields_follow_the_existing_descriptor():
    from selfocc_b200 import _lib
    names = [f[0] for f in _lib.ObjectiveDesc._fields_]
    assert names[-4:] == ['workspace_bytes', 'second_grad', 'second_grad_mean', 'grad_second_grad_mean']
    d = _lib.ObjectiveDesc()
    assert d.second_grad == 0 and not d.second_grad_mean and not d.grad_second_grad_mean      # zero-initialised = off
    assert _lib.ObjectiveDesc.second_grad.offset >= _lib.ObjectiveDesc.workspace_bytes.offset + 8


def test_second_grad_calls_without_rays_return_ok(lib):
    assert _fwd(lib, _objective(second_grad=1, second_grad_mean=16)) == 0
    assert _fwd(lib, _objective(reproj_mode=-1, eikonal=0, second_grad=1, second_grad_mean=16), stats=None, mean=None) == 0
    assert _bwd(lib, _objective(second_grad=1, grad_second_grad_mean=16)) == 0
    assert _bwd(lib, _objective(second_grad=1)) == 0                         # NULL cotangent = 0


@pytest.mark.parametrize('ob, rd, code', [
    (dict(second_grad=2, second_grad_mean=16), None, INVALID),
    (dict(second_grad=-1), None, INVALID),
    (dict(second_grad=1), None, INVALID),                                     # no output
    (dict(second_grad=1, second_grad_mean=18), None, INVALID),                # misaligned output
    (dict(second_grad=1, second_grad_mean=16, workspace=0), None, INVALID),
    (dict(second_grad=1, second_grad_mean=16, workspace=20), None, INVALID),  # not 8-byte aligned
    # both means: 16 bytes per ray
    (dict(second_grad=1, second_grad_mean=16, workspace_bytes=8 * 4), dict(ray_count=4), INVALID),
    (dict(second_grad=1, second_grad_mean=16, workspace_bytes=16 * 4 - 8), dict(ray_count=4), INVALID),
    # the second-grad mean alone: 8 bytes per ray
    (dict(reproj_mode=-1, eikonal=0, second_grad=1, second_grad_mean=16, workspace_bytes=8 * 4 - 8), dict(ray_count=4), INVALID),
])
def test_forward_refuses_bad_second_grad_arguments(lib, ob, rd, code):
    kw = dict(stats=None, mean=None) if ob.get('reproj_mode') == -1 else {}
    assert _fwd(lib, _objective(**ob), rd=rd, **kw) == code


@pytest.mark.parametrize('ob', [dict(second_grad=2), dict(second_grad=1, grad_second_grad_mean=18)])
def test_backward_refuses_bad_second_grad_arguments(lib, ob):
    assert _bwd(lib, _objective(**ob)) == INVALID


def test_render_train_objective_function_orders_the_new_output_last():
    from selfocc_b200 import ops
    assert ops.RenderTrainObjectiveFunction.ORDER[-2:] == ('eikonal_mean', 'second_grad_mean')
    d = ops.RenderTrainObjectiveFunction._desc(dict(mode=None, eikonal=True, second_grad=True))
    assert d.second_grad == 1 and d.eikonal == 1 and d.reproj_mode == -1
    assert ops.RenderTrainObjectiveFunction._desc(dict(mode=None, eikonal=True)).second_grad == 0


# ------------------------------------------------------------------------------------------------ fp64 oracle
def test_oracle_second_grad_of_a_trilinear_monomial_field():
    """vol = h w + 2 h z - 3 w z: d2/dh dw = 1, d2/dh dz = 2, d2/dw dz = -3 in every cell; with slopes (kh, kw, kd) the
    metre Hessian entries are Hxy = kw kh, Hyz = 2 kh kd, Hxz = -3 kw kd.  Points whose cell leaves the volume see zeros."""
    from oracle.second_grad import second_grad_ref
    H, W, Z = 5, 6, 4
    h, w, z = torch.meshgrid(torch.arange(H), torch.arange(W), torch.arange(Z), indexing='ij')
    vol = (h * w + 2 * h * z - 3 * w * z).double()
    g = torch.Generator().manual_seed(0)
    pts = torch.rand(50, 3, generator=g, dtype=torch.float64) * torch.tensor([H - 1., W - 1., Z - 1.])
    k = torch.tensor([[0.5, 2.0, 1.5]], dtype=torch.float64).expand(50, 3)
    x = second_grad_ref(vol, pts, k)
    kh, kw, kd = 0.5, 2.0, 1.5
    Hxy, Hyz, Hxz = kw * kh, 2 * kh * kd, -3 * kw * kd
    assert torch.allclose(x, torch.tensor([Hxy + Hxz, Hxy + Hyz, Hxz + Hyz], dtype=torch.float64).expand(50, 3))
    far = torch.tensor([[-3.5, 2.2, 1.1], [1.0, 2.0, Z + 0.5]], dtype=torch.float64)
    assert torch.equal(second_grad_ref(vol, far, k[:2]), torch.zeros(2, 3, dtype=torch.float64))


def test_oracle_second_grad_mean_gradient_is_the_derivative_of_the_mean():
    from oracle.second_grad import second_grad_mean_ref, axis_slopes
    g = torch.Generator().manual_seed(1)
    vol = torch.randn(6, 5, 4, generator=g, dtype=torch.float64)
    pts = torch.rand(200, 3, generator=g, dtype=torch.float64) * torch.tensor([7.0, 6.0, 5.0]) - 1.0     # some leave the volume
    k = axis_slopes(pts, [(0.0, 3.0, 0.5, 0.25), (0.0, 10.0, 2.0, 0.0), (0.0, 10.0, 1.5, 0.0)])
    assert set(k[:, 0].tolist()) == {0.5, 0.25} and set(k[:, 1].tolist()) == {2.0}
    mean, grad, bound, n_amb = second_grad_mean_ref(vol, pts, k, g_mean=0.7, chunk=64)
    assert n_amb == 0 and bound.abs().max() == 0
    d = torch.randn(vol.shape, generator=g, dtype=torch.float64)
    eps = 1e-6
    hi = second_grad_mean_ref(vol + eps * d, pts, k)[0]
    lo = second_grad_mean_ref(vol - eps * d, pts, k)[0]
    assert abs(0.7 * (hi - lo) / (2 * eps) - (grad * d).sum()) <= 1e-6 * abs((grad * d).sum())
