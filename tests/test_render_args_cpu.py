"""Return codes of the render entry points for bad and edge arguments.

Every case checks its arguments before any CUDA call: the ray count is 0 throughout (or the ray range is invalid), so no
kernel is ever launched and this runs on a CPU-only box.  The table pins, for each entry point, which code comes back,
including which of SO_ERR_INVALID_ARG (-1) and SO_ERR_UNSUPPORTED (-2) wins when both apply."""
import ctypes as C

import pytest

ENTRIES = ('infer', 'packed', 'train_fwd', 'train_bwd', 'probe')
ONE = C.c_void_p(16)       # non-null, 16-byte aligned dummy (never dereferenced on these paths)


def _desc(H=9, W=9, Z=5, zpitch=8, n_feat=0, feat_pitch=0, outer_ring=False):
    from selfocc_b200 import _lib
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = H, W, Z, zpitch, n_feat, feat_pitch
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 1.0, 4.0
        if outer_ring:
            d.axis[i].range1, d.axis[i].size1 = 2.0, 2.0
    return d


def _rays(**kw):
    from selfocc_b200 import _lib
    rd = _lib.RayDesc()
    rd.n_cam, rd.rays_per_cam, rd.nx, rd.ny, rd.ray_begin, rd.ray_count = 1, 4, 2, 2, 0, 0
    for k, v in kw.items():
        setattr(rd, k, v)
    return rd


def _params(**kw):
    from selfocc_b200 import _lib
    pr = _lib.RenderParams()
    pr.num_samples, pr.inv_s, pr.cos_anneal, pr.anchor_mid, pr.sh_act, pr.bkgd_mode = 64, 20.0, 1.0, 1, 0, 0
    for k, v in kw.items():
        setattr(pr, k, v)
    return pr


# operands of one call; every entry point takes the ones it has.  rgb / sem stand for the colour / semantic outputs of
# the forwards and for their cotangents in the backward.
DEFAULTS = dict(vol_sdf=ONE, vol_feat=None, desc='d0', cam=ONE, pix=None, rd={}, pr={}, bkgd=None, ws=ONE, rgb=None,
                sem=None, pack=None, dbg=None, pair=None, g_vol_sdf=ONE, g_vol_feat=None, grid=ONE)

DESCS = dict(d0=dict(), d3=dict(n_feat=3, feat_pitch=4), d24=dict(n_feat=24, feat_pitch=24), d40=dict(n_feat=40, feat_pitch=40),
             ring=dict(outer_ring=True), bad=dict(zpitch=4), badfeat=dict(n_feat=3, feat_pitch=3),
             big=dict(H=40000, W=40000, Z=2, zpitch=8), none=None)


def _call(lib, entry, case):
    a = dict(DEFAULTS, **case)
    d = None if DESCS[a['desc']] is None else _desc(**DESCS[a['desc']])
    rd = None if a['rd'] is None else _rays(**a['rd'])
    pr = None if a['pr'] is None else _params(**a['pr'])
    dp, rp, pp = (None if x is None else C.byref(x) for x in (d, rd, pr))
    N = None
    if entry == 'infer':
        return lib.so_render_infer(a['vol_sdf'], a['vol_feat'], dp, a['cam'], a['pix'], rp, pp, a['bkgd'], ONE, N, N, N, N,
                                   a['rgb'], a['sem'], a['ws'], N)
    if entry == 'packed':
        return lib.so_render_infer_packed(a['vol_sdf'], a['vol_feat'], dp, a['pack'], a['cam'], a['pix'], rp, pp, a['bkgd'], ONE,
                                          N, N, N, N, a['rgb'], a['sem'], a['ws'], a['dbg'], N)
    if entry == 'train_fwd':
        return lib.so_render_train_forward(a['vol_sdf'], a['vol_feat'], dp, a['cam'], a['pix'], rp, pp, N, a['bkgd'], ONE, N, N,
                                           a['rgb'], a['sem'], N, N, N, N, N, N, a['ws'], a['pair'], N)
    if entry == 'train_bwd':
        return lib.so_render_train_backward(a['vol_sdf'], a['vol_feat'], dp, a['cam'], a['pix'], rp, pp, N, a['bkgd'], ONE, N,
                                            a['rgb'], a['sem'], N, N, N, a['g_vol_sdf'], a['g_vol_feat'], N, a['ws'], N)
    return lib.so_render_train_probe(dp, a['cam'], a['pix'], rp, pp, N, a['grid'], N)


FEAT3 = dict(desc='d3', vol_feat=ONE, g_vol_feat=ONE)
SEM24 = dict(desc='d24', vol_feat=ONE, g_vol_feat=ONE, rgb=ONE, sem=ONE)
SEM40 = dict(desc='d40', vol_feat=ONE, g_vol_feat=ONE, rgb=ONE, sem=ONE)
BAD_RAYS = dict(rd=dict(ray_begin=5))

# case -> operands; expected codes per entry point in ENTRIES order
CASES = {
    'ray_count_0': (dict(), (0, 0, 0, 0, 0)),
    'null_vol_sdf': (dict(vol_sdf=None), (-1, -1, -1, -1, 0)),
    'null_cameras': (dict(cam=None), (-1, -1, -1, -1, -1)),
    'null_rays': (dict(rd=None), (-1, -1, -1, -1, -1)),
    'null_params': (dict(pr=None), (-1, -1, -1, -1, -1)),
    'null_workspace': (dict(ws=None), (-1, -1, -1, -1, 0)),
    'null_probe_grid': (dict(grid=None), (0, 0, 0, 0, -1)),
    'null_volume_desc': (dict(desc='none'), (-1, -1, -1, -1, -1)),
    'zpitch_below_Z': (dict(desc='bad'), (-1, -1, -1, -1, -1)),
    'feat_pitch_below_n_feat': (dict(desc='badfeat'), (-1, -1, -1, -1, -1)),
    'oversized_volume': (dict(desc='big'), (-2, -2, -2, -2, -2)),
    'no_cameras': (dict(rd=dict(n_cam=0)), (-1, -1, -1, -1, -1)),
    'no_rays_per_camera': (dict(rd=dict(rays_per_cam=0)), (-1, -1, -1, -1, -1)),
    'grid_not_rays_per_cam': (dict(rd=dict(nx=3)), (-1, -1, -1, -1, -1)),
    'grid_not_rays_per_cam_with_pixels': (dict(rd=dict(nx=3), pix=ONE), (0, 0, 0, 0, 0)),
    'no_grid_width': (dict(rd=dict(nx=0, ny=4)), (-1, -1, -1, -1, -1)),
    'negative_ray_begin': (dict(rd=dict(ray_begin=-1)), (-1, -1, -1, -1, -1)),
    'rays_past_the_end': (BAD_RAYS, (-1, -1, -1, -1, -1)),
    'negative_ray_count': (dict(rd=dict(ray_count=-1)), (-1, -1, -1, -1, -1)),
    'S_0': (dict(pr=dict(num_samples=0)), (-1, -1, -1, -1, -1)),
    'S_1': (dict(pr=dict(num_samples=1)), (0, 0, 0, 0, 0)),
    'S_48': (dict(pr=dict(num_samples=48)), (0, 0, 0, 0, 0)),
    'S_257': (dict(pr=dict(num_samples=257)), (0, 0, -2, -2, -2)),
    'rgb_without_features': (dict(rgb=ONE), (-1, -1, -1, -1, 0)),
    'rgb_without_feature_volume': (dict(FEAT3, vol_feat=None, rgb=ONE), (-1, -1, -1, -1, 0)),
    'rgb': (dict(FEAT3, rgb=ONE), (0, 0, 0, 0, 0)),
    'rgb_without_feature_gradient': (dict(FEAT3, rgb=ONE, g_vol_feat=None), (0, 0, 0, -1, 0)),
    'sem_with_3_channels': (dict(FEAT3, rgb=ONE, sem=ONE), (-1, -1, -1, -1, 0)),
    'sem_without_feature_volume': (dict(SEM24, vol_feat=None), (-1, -1, -1, -1, 0)),
    'sem_24': (SEM24, (0, 0, 0, 0, 0)),
    'sem_without_rgb': (dict(SEM24, rgb=None), (-1, -1, 0, 0, 0)),
    'sem_37_classes': (SEM40, (-2, -2, -2, -2, 0)),
    'random_background_without_colours': (dict(FEAT3, rgb=ONE, pr=dict(bkgd_mode=2)), (-1, -1, -1, -1, 0)),
    'random_background_with_colours': (dict(FEAT3, rgb=ONE, bkgd=ONE, pr=dict(bkgd_mode=2)), (0, 0, 0, 0, 0)),
    'random_background_depth_only': (dict(pr=dict(bkgd_mode=2)), (0, 0, 0, 0, 0)),
    'bkgd_mode_3': (dict(pr=dict(bkgd_mode=3)), (-1, -1, -1, -1, 0)),
    'bkgd_mode_negative': (dict(pr=dict(bkgd_mode=-1)), (-1, -1, -1, -1, 0)),
    'sh_act_2': (dict(pr=dict(sh_act=2)), (-1, -1, -1, -1, 0)),
    'sigmoid_colour': (dict(FEAT3, rgb=ONE, pr=dict(sh_act=1)), (0, 0, 0, 0, 0)),
    'misaligned_pair_scratch': (dict(pair=C.c_void_p(20)), (0, 0, -1, 0, 0)),
    'pair_scratch': (dict(pair=ONE), (0, 0, 0, 0, 0)),
    'no_volume_gradient': (dict(g_vol_sdf=None), (0, 0, 0, -1, 0)),
    'pack': (dict(pack=ONE), (0, 0, 0, 0, 0)),
    'pack_rgb': (dict(FEAT3, pack=ONE, rgb=ONE), (0, 0, 0, 0, 0)),
    'pack_rgb_without_feature_volume': (dict(FEAT3, pack=ONE, rgb=ONE, vol_feat=None), (-1, 0, -1, -1, 0)),
    'pack_sem': (dict(SEM24, pack=ONE), (0, 0, 0, 0, 0)),
    'pack_outer_ring': (dict(desc='ring', pack=ONE), (0, 0, 0, 0, 0)),
    'probe_grid_without_pack': (dict(dbg=ONE), (0, -2, 0, 0, 0)),
    'probe_grid': (dict(pack=ONE, dbg=ONE), (0, 0, 0, 0, 0)),
    'probe_grid_S_48': (dict(pack=ONE, dbg=ONE, pr=dict(num_samples=48)), (0, -2, 0, 0, 0)),
    'probe_grid_cos_anneal': (dict(pack=ONE, dbg=ONE, pr=dict(cos_anneal=0.5)), (0, -2, 0, 0, 0)),
    # several checks fail at once
    'probe_grid_S_0': (dict(pack=ONE, dbg=ONE, pr=dict(num_samples=0)), (-1, -2, -1, -1, -1)),
    'probe_grid_bad_volume': (dict(pack=ONE, dbg=ONE, desc='bad'), (-1, -1, -1, -1, -1)),
    'probe_grid_bad_rays': (dict(pack=ONE, dbg=ONE, rd=dict(ray_begin=5)), (-1, -1, -1, -1, -1)),
    'probe_grid_bkgd_mode_3': (dict(pack=ONE, dbg=ONE, pr=dict(bkgd_mode=3)), (-1, -1, -1, -1, 0)),
    'oversized_volume_null_cameras': (dict(desc='big', cam=None), (-1, -1, -1, -1, -1)),
    'oversized_volume_bad_rays': (dict(BAD_RAYS, desc='big'), (-2, -2, -2, -2, -2)),
    'sem_37_classes_bad_rays': (dict(SEM40, **BAD_RAYS), (-1, -1, -2, -2, -1)),
    'sem_37_classes_without_rgb': (dict(SEM40, rgb=None), (-1, -1, -2, -2, 0)),
    'sem_37_classes_bkgd_mode_3': (dict(SEM40, pr=dict(bkgd_mode=3)), (-2, -2, -2, -2, 0)),
    'sem_37_classes_S_0': (dict(SEM40, pr=dict(num_samples=0)), (-1, -1, -1, -1, -1)),
    'S_257_bad_rays': (dict(BAD_RAYS, pr=dict(num_samples=257)), (-1, -1, -2, -2, -2)),
    'S_257_rgb_without_features': (dict(rgb=ONE, pr=dict(num_samples=257)), (-1, -1, -2, -2, -2)),
    'S_257_bkgd_mode_3': (dict(pr=dict(num_samples=257, bkgd_mode=3)), (-1, -1, -2, -2, -2)),
    'random_background_without_colours_bad_rays': (dict(FEAT3, rgb=ONE, pr=dict(bkgd_mode=2), **BAD_RAYS), (-1, -1, -1, -1, -1)),
    'misaligned_pair_scratch_oversized_volume': (dict(pair=C.c_void_p(20), desc='big'), (-2, -2, -1, -2, -2)),
    'no_volume_gradient_null_cameras': (dict(g_vol_sdf=None, cam=None), (-1, -1, -1, -1, -1)),
}


@pytest.fixture(scope='module')
def lib():
    import os
    from selfocc_b200 import _lib, build
    if not os.environ.get('SELFOCC_B200_LIB'):
        build.build()
    return _lib.load()


@pytest.mark.parametrize('case', sorted(CASES))
def test_render_entry_point_return_codes(lib, case):
    operands, expected = CASES[case]
    assert (operands.get('rd') or {}).get('ray_count', 0) <= 0      # a case that passed every check must not launch
    got = tuple(_call(lib, entry, operands) for entry in ENTRIES)
    assert got == expected, dict(zip(ENTRIES, got))
