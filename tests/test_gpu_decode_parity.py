"""GPU parity of the TPV decode (B5: so_tpv_decode / so_tpv_decode_rows and the slab backward behind
ops.TPVDecodeFunction) against the fp64 oracle evaluated slab by slab on the device (oracle/decode_parity.py):

  * forward on EVERY voxel and channel at the shipped configs' volume geometry, both kernels, into NaN-filled buffers;
  * the persistent wgmma kernel's tile loop, masks and instantiations at volumes chosen from its tile arithmetic;
  * row slabs (so_tpv_decode_rows) into NaN-filled buffers;
  * inputs that cover the whole softplus domain, with the activation and sigmoid errors reported per pre-activation bucket;
  * the backward at shipped geometry with the shipped slab height: per tensor, and per channel / row / column / entry
    relative to that slice's own magnitude, on standard inputs and on inputs with channels shifted far negative.

Pad contract of the C entry points (include/selfocc_b200.h): sdf pads z in [Z, zpitch) are written as 0 for the rows of
the launch; feature pad channels [n_feat, feat_pitch) are never written (ops.tpv_decode zeroes them itself).
"""
import ctypes as C
import json
import os

import pytest
import torch

from selfocc_b200.mapping import GridMeterMapping

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(ROOT, 'golden', 'reference_model_cfgs.json')))
NAN = float('nan')

# name -> (config, decoded feature channels, expected (H, W, Z, zpitch, feat_pitch))
SHIPPED = {
    'nuScenes_depth': ('nuscenes/nuscenes_depth.py', 0, (257, 257, 31, 32, 0)),
    'nuScenes_novel_depth': ('nuscenes/nuscenes_novel_depth.py', 3, (257, 257, 31, 32, 4)),
    'nuScenes_occ': ('nuscenes/nuscenes_occ.py', 24, (257, 257, 25, 32, 24)),
    'KITTI_occ': ('kitti/kitti_occ.py', 3, (257, 257, 33, 40, 4)),              # h_half
    'KITTI_raw_depth': ('kitti_raw/kitti_raw_depth.py', 0, (257, 257, 33, 40, 0)),
    # not shipped: feature counts whose pad is 3 and 1 channels, second-layer width 6 and 8 (the NOUT = 32 instantiation)
    'nuScenes_geometry_5_features': ('nuscenes/nuscenes_depth.py', 5, (257, 257, 31, 32, 8)),
    'nuScenes_geometry_7_features': ('nuscenes/nuscenes_depth.py', 7, (257, 257, 31, 32, 8)),
}
# existing bars of tests/test_gpu_render.py::test_tpv_decode_matches_oracle
SDF_BAR = 2e-5                      # times max(1, |sdf| max)
FEAT_ATOL, FEAT_RTOL = 5e-5, 1e-5


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _desc(H, W, Z, n_feat):
    """Volume descriptor with the pitches GridMeterMapping.volume_desc gives; the decode reads sizes and pitches only."""
    from selfocc_b200 import _lib
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = H, W, Z, (Z + 7) // 8 * 8, n_feat, (n_feat + 3) // 4 * 4
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 1.0, 1.0
    return d


def _shipped_desc(name):
    cfg, n_feat, expect = SHIPPED[name]
    d = GridMeterMapping(**CFGS[cfg]['head']['mapping_args']).volume_desc(n_feat)
    assert (d.H, d.W, d.Z, d.zpitch, d.feat_pitch) == expect
    return d


def _inputs(d, Cc, seed, scale=1.0):
    """Planes N(0, scale) and the MLP of synth.random_mlp (what every other decode test draws), on the device."""
    from selfocc_b200 import synth
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    planes = [(scale * torch.randn(n, Cc, generator=g)).to(dev) for n in (d.H * d.W, d.Z * d.H, d.W * d.Z)]
    return planes, [t.to(dev) for t in synth.random_mlp(Cc, 1 + d.n_feat, seed=seed)]


def _oracle(planes, mlp, d):
    from oracle import decode_parity as dp
    return dp.decode_slabwise(*[p.double() for p in planes], (d.H, d.W, d.Z), *[t.double() for t in mlp])


def _launch(planes, mlp, d, simt=False, rows=None, out=None):
    """so_tpv_decode_rows through the C ABI into NaN-filled (or the given) full-size buffers."""
    from selfocc_b200 import _lib, ops
    lib = _lib.load()
    dev = planes[0].device
    if out is None:
        out = (torch.full((d.H, d.W, d.zpitch), NAN, device=dev),
               torch.full((d.H, d.W, d.Z, d.feat_pitch), NAN, device=dev) if d.n_feat else None)
    h0, hc = (0, d.H) if rows is None else rows
    lib.so_tpv_decode_force_simt(int(simt))
    try:
        _lib.check(lib.so_tpv_decode_rows(*map(ops._p, planes), planes[0].shape[-1], *map(ops._p, mlp),
                                          C.byref(d), h0, hc, ops._p(out[0]), ops._p(out[1]), ops._stream()), 'so_tpv_decode_rows')
    finally:
        lib.so_tpv_decode_force_simt(0)
    return out


def _same_bits(a, b):
    return a is b or torch.equal(a.view(torch.int32), b.view(torch.int32))


def _check_volume(out, ref, d, rows=None, scale=1.0):
    """Every voxel and channel of rows [h0, h0 + hc) against the oracle at ``scale`` times the bars; sdf pads of those rows
    exactly 0, feature pad channels untouched (NaN), every other row untouched (NaN), pads included.
    Returns (sdf max abs err, feature max abs err)."""
    vs, vf = out
    h0, hc = (0, d.H) if rows is None else rows
    inside = torch.zeros(d.H, dtype=torch.bool, device=vs.device)
    inside[h0:h0 + hc] = True
    assert torch.isnan(vs[~inside]).all(), 'sdf rows outside the launch were written'
    assert (vs[inside][..., d.Z:] == 0).all(), 'sdf pads are not exactly 0'
    if not hc:
        assert vf is None or torch.isnan(vf).all()
        return 0.0, 0.0
    got, want = vs[inside][..., :d.Z].double(), ref[inside][..., 0]
    assert not torch.isnan(got).any(), '%d sdf voxels were not written' % int(torch.isnan(got).sum())
    e_sdf = float((got - want).abs().max())
    assert e_sdf <= scale * SDF_BAR * max(1.0, float(want.abs().max())), 'sdf max abs err %.3e' % e_sdf
    e_feat = 0.0
    if d.n_feat:
        assert torch.isnan(vf[~inside]).all(), 'feature rows outside the launch were written'
        assert torch.isnan(vf[inside][..., d.n_feat:]).all(), 'feature pad channels were written'
        got, want = vf[inside][..., :d.n_feat].double(), ref[inside][..., 1:]
        assert not torch.isnan(got).any(), '%d feature entries were not written' % int(torch.isnan(got).sum())
        err = (got - want).abs()
        e_feat = float(err.max())
        worst = float((err / (FEAT_ATOL + FEAT_RTOL * want.abs())).max())
        assert worst <= scale, 'features miss atol %.0e + rtol %.0e by a factor %.2f (max abs err %.3e)' % (FEAT_ATOL, FEAT_RTOL, worst, e_feat)
    return e_sdf, e_feat


def _check_pair(tc, simt, ref, d):
    """wgmma against SIMT on the same inputs: each is within one bar of the oracle, so they are within two of each other."""
    a, b = tc[0][..., :d.Z].double(), simt[0][..., :d.Z].double()
    assert float((a - b).abs().max()) <= 2 * SDF_BAR * max(1.0, float(ref[..., 0].abs().max()))
    if d.n_feat:
        a, b = tc[1][..., :d.n_feat].double(), simt[1][..., :d.n_feat].double()
        assert float(((a - b).abs() / (FEAT_ATOL + FEAT_RTOL * ref[..., 1:].abs())).max()) <= 2.0


# ---- 1. forward, every voxel, shipped geometry -----------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('name', list(SHIPPED))
def test_forward_every_voxel_at_shipped_geometry(name):
    _dev()
    from selfocc_b200 import ops
    d = _shipped_desc(name)
    planes, mlp = _inputs(d, 96, seed=11)
    ref = _oracle(planes, mlp, d)
    out = {}
    for simt in (False, True):
        out[simt] = _launch(planes, mlp, d, simt)
        e = _check_volume(out[simt], ref, d)
        print('%s forward (%s): sdf max abs err %.3e (|sdf| max %.2f), features max abs err %.3e'
              % (name, 'simt' if simt else 'wgmma', e[0], float(ref[..., 0].abs().max()), e[1]))
    _check_pair(out[False], out[True], ref, d)
    for simt in (False, True):
        again = _launch(planes, mlp, d, simt)
        assert _same_bits(again[0], out[simt][0]) and (not d.n_feat or _same_bits(again[1], out[simt][1])), 'two launches differ'
    # the torch front end allocates the buffers and zeroes the feature pad channels; same kernel, same bits elsewhere
    vs, vf = ops.tpv_decode(*planes, *mlp, d)
    assert torch.equal(vs, out[False][0])
    if d.n_feat:
        assert torch.equal(vf[..., :d.n_feat], out[False][1][..., :d.n_feat]) and (vf[..., d.n_feat:] == 0).all()


# ---- 2. the persistent loop and the instantiations ---------------------------------------------------------------------------
# The wgmma kernel decodes tiles of 128 consecutive (w, z) voxels of one h row: tiles_per_row = ceil(W Z / 128), tiles =
# tiles_per_row H, grid = min(tiles, SMs), CTA b takes tiles b, b + grid, ...; the stage ring (2-4 stages) carries its index and
# phase bit across tiles while a tile is C / 32 atoms (3 atoms on 4 stages at C = 96: the ring wraps inside every tile but
# the first).  Consumer warpgroup 0 owns voxels 0-63 of a tile, warpgroup 1 voxels 64-127; a thread holds rows r and r + 8
# of a 16-row fragment.  Each geometry is (H as a function of the SM count, W, Z, what W Z mod 128 leaves in the last tile).
TILE_GEOMETRIES = {
    # two tiles per row, H = SMs + 1: 2 SMs + 2 tiles, every CTA takes two or three, the count is not a multiple of the grid
    'wz_129': (lambda sms: sms + 1, 43, 3),      # 1 voxel in the last tile: row 0 of a fragment pair valid, row 8 masked
    'wz_159': (lambda sms: sms + 1, 53, 3),      # 31: the mask boundary inside warpgroup 0, inside a fragment pair's second row
    'wz_192': (lambda sms: sms + 1, 64, 3),      # 64: warpgroup 1 of the last tile entirely masked
    'wz_193_z1': (lambda sms: sms + 1, 193, 1),  # 65: one voxel of warpgroup 1; Z = 1 (w = v, z = 0)
    'wz_255': (lambda sms: sms + 1, 51, 5),      # 127: only the last voxel masked
    # one partial tile per row (W Z = 63 < 128), Z = 7: (v + 1/2) / 7 by reciprocal; 2 SMs + 3 tiles
    'wz_63_z7': (lambda sms: 2 * sms + 3, 9, 7),
    # a single h row of 10 tiles (88 voxels in the last): grid = tiles, no second tile
    'h_1': (lambda sms: 1, 40, 31),
}
CHANNELS = (32, 64, 96, 128)
N_OUT = (1, 2, 4, 5, 25, 32)       # instantiations NOUT = 1 | 4 | 32 cover n_out 1 | 2-4 | 5-32: both ends of each


def _dec_stages(Cc, n_out):
    """dec_smem of decode.cu: ring stages left beside the resident W1 hi / lo (below 2 the SIMT kernel takes over)."""
    fixed = 2 * (Cc // 32) * Cc * 128 + n_out * Cc * 4 + Cc * 4 + 128 + 256
    return min(4, (227 * 1024 - 1024 - fixed) // (2 * 128 * 128))


@gpu
@pytest.mark.parametrize('geom', list(TILE_GEOMETRIES))
def test_forward_tile_loop_masks_and_instantiations(geom):
    dev = _dev()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    fH, W, Z = TILE_GEOMETRIES[geom]
    H = fH(sms)
    tiles = -(-W * Z // 128) * H
    if geom != 'h_1':
        assert tiles > 2 * sms and tiles % sms != 0
    worst = [0.0, 0.0]
    for Cc in CHANNELS:
        for n_out in N_OUT:
            d = _desc(H, W, Z, n_out - 1)
            planes, mlp = _inputs(d, Cc, seed=Cc + n_out)
            ref = _oracle(planes, mlp, d)
            tc, simt = _launch(planes, mlp, d, False), _launch(planes, mlp, d, True)
            for out in (tc, simt):
                e = _check_volume(out, ref, d)
                worst = [max(a, b) for a, b in zip(worst, e)]
            _check_pair(tc, simt, ref, d)
            # the two kernels round differently (3xTF32 products, another summation order): equal bits would mean the
            # launch fell back to the SIMT kernel.  Every listed size leaves the ring at least 2 stages (C = 128 with
            # n_out = 32 exactly 2), so the wgmma kernel is what ran.
            assert _dec_stages(Cc, n_out) >= 2 and not _same_bits(tc[0], simt[0])
    assert _dec_stages(128, 32) == 2 and _dec_stages(96, 4) == 4
    print('%s: H %d W %d Z %d, %d tiles on %d SMs, %d (C, n_out) pairs x 2 kernels: sdf max abs err %.3e, features %.3e'
          % (geom, H, W, Z, tiles, sms, len(CHANNELS) * len(N_OUT), *worst))


def test_unsupported_widths_are_refused_before_any_launch():
    """A second layer wider than 32 outputs and a channel count other than 32 / 64 / 96 / 128 return SO_ERR_UNSUPPORTED (-2)
    before any CUDA call, also when the volume has sdf pads to zero; so this runs without a GPU, on never-dereferenced dummy
    pointers.  Where a GPU is present the outputs are real buffers."""
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    one, N = C.c_void_p(16), None
    for Z in (8, 31):                                  # zpitch == Z, and a padded volume
        wide, d = _desc(9, 9, Z, 32), _desc(9, 9, Z, 3)          # n_out = 33; n_out = 4
        vs = vf = one
        if torch.cuda.is_available():
            bufs = (torch.zeros(9, 9, d.zpitch, device='cuda'), torch.zeros(9, 9, Z, 32, device='cuda'))
            vs, vf = (C.c_void_p(t.data_ptr()) for t in bufs)
        assert lib.so_tpv_decode(one, one, one, 96, one, one, one, one, C.byref(wide), vs, vf, N) == -2
        for Cc in (48, 16, 160, 0, 100):
            assert lib.so_tpv_decode(one, one, one, Cc, one, one, one, one, C.byref(d), vs, vf, N) == -2, Cc
            assert lib.so_tpv_decode_rows(one, one, one, Cc, one, one, one, one, C.byref(d), 2, 3, vs, vf, N) == -2, Cc
    assert lib.so_tpv_decode(one, one, one, 96, one, one, one, one, C.byref(_desc(9, 9, 8, 3)), one, N, N) == -1   # no feature volume


@gpu
@pytest.mark.parametrize('simt', [False, True])
def test_row_slabs_write_their_rows_only_and_tile_the_whole_launch(simt):
    """so_tpv_decode_rows at the nuScenes novel-depth volume: ragged slabs, a one-row first and last slab, an empty one."""
    _dev()
    d = _shipped_desc('nuScenes_novel_depth')
    planes, mlp = _inputs(d, 96, seed=12)
    ref = _oracle(planes, mlp, d)
    whole = _launch(planes, mlp, d, simt)
    _check_volume(whole, ref, d)
    union = None
    for rows in ((100, 0), (0, 1), (1, 32), (33, 223), (256, 1)):
        _check_volume(_launch(planes, mlp, d, simt, rows=rows), ref, d, rows=rows)
        union = _launch(planes, mlp, d, simt, rows=rows, out=union)
    assert _same_bits(union[0], whole[0]) and _same_bits(union[1], whole[1])


# ---- 3. the activation's whole domain ----------------------------------------------------------------------------------------
def _wide_inputs(d, Cc, seed):
    """Planes whose sum f covers softplus's whole domain, and a first-layer bias to match:
    channels 0-15 carry N(0, 8) planes (f ~ N(0, 14): beyond +-40, through the threshold 20 on both sides);
    channel 16: f = 0 exactly on h row 0; 17: f = +20 and 18: f = -20 exactly on h row 1; 19: every plane entry a denormal
    (f = 6e-39: the library is built with -ftz and reads it as 0, the oracle keeps it; softplus differs by 3e-39, far below
    any bar, so the one comparison accepts both); 20: shifted to -10; 21: shifted to +30; the rest N(0, 1) like every other test.
    b1 entries at -12, -6, 0 and +25."""
    planes, mlp = _inputs(d, Cc, seed)
    hw, zh, wz = planes[0].view(d.H, d.W, Cc), planes[1].view(d.Z, d.H, Cc), planes[2].view(d.W, d.Z, Cc)
    for p in (hw, zh, wz):
        p[..., :16] *= 8.0
        p[..., 16:20] = 0.0
        p[..., 19] = 2e-39
        p[..., 20:22] *= 0.5
    hw[1, :, 17], hw[1, :, 18] = 20.0, -20.0
    hw[2:, :, 16:19] = torch.randn(d.H - 2, d.W, 3, generator=torch.Generator().manual_seed(seed)).to(hw.device)
    hw[..., 20] -= 10.0
    hw[..., 21] += 30.0
    b1 = mlp[1]
    b1[0:8], b1[8:16], b1[16:24], b1[24:32] = -12.0, -6.0, 0.0, 25.0
    return planes, mlp


def _print_buckets(tag, rows):
    from oracle import decode_parity as dp
    print('  %s: ' % tag + ' | '.join('[%g, %g) n %d abs %.1e rel %.1e' % (lo, hi, n, a, r) for (lo, hi), (n, a, r) in zip(dp.BUCKETS, rows)))


# relative bars per bucket of oracle/decode_parity.py:BUCKETS.  Below -16 the fp32 rounding of the pre-activation itself is
# 1 ulp(|x|) ~ 2e-6 |x| / 16 relative to exp(x); it is reported and held to 3e-5.  On the negative side, where the value is
# below ln 2, the absolute error is held to 1e-6 as well.
ACT_REL_BARS = (3e-5, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5, 1e-5)


def _assert_buckets(tag, rows, need=range(7)):
    _print_buckets(tag, rows)
    for i, ((n, a, r), bar) in enumerate(zip(rows, ACT_REL_BARS)):
        assert n > 0 or i not in need, '%s: no element in bucket %d' % (tag, i)
        assert r <= bar and (i > 4 or a <= 1e-6), '%s: bucket %d abs %.2e rel %.2e' % (tag, i, a, r)


@gpu
def test_forward_over_the_whole_activation_domain():
    _dev()
    d = _desc(40, 48, 13, 3)
    planes, mlp = _wide_inputs(d, 96, seed=13)
    from oracle import decode_parity as dp
    f = dp.preactivation(*[p.double() for p in planes], (d.H, d.W, d.Z), 0, d.H)
    assert f.min() < -40 and f.max() > 40 and (f[0, ..., 16] == 0).all() and (f[1, ..., 17] == 20).all() and (f[1, ..., 18] == -20).all()
    assert 0 < f[..., 19].max() < 1e-38
    ref = _oracle(planes, mlp, d)
    tc, simt = _launch(planes, mlp, d, False), _launch(planes, mlp, d, True)
    for name, out in (('wgmma', tc), ('simt', simt)):
        e = _check_volume(out, ref, d)
        print('wide inputs (%s): sdf max abs err %.3e (|sdf| max %.2f), features max abs err %.3e (|f| max %.2f)'
              % (name, e[0], float(ref[..., 0].abs().max()), e[1], float(ref[..., 1:].abs().max())))
    _check_pair(tc, simt, ref, d)


@gpu
def test_backward_activations_are_accurate_relative_to_their_value():
    """The three element-wise kernels of the slab backward through the C ABI: a0 = softplus(f) of so_tpv_decode_bwd_features
    and sigmoid(f) as so_tpv_decode_bwd_input forms it from a0, on the wide planes; softplus(z) and sigmoid(z) of
    so_tpv_decode_bwd_hidden on a grid of z.  Error against fp64 per bucket of the argument, absolute and relative."""
    dev = _dev()
    from oracle import decode_parity as dp
    from selfocc_b200 import _lib, ops
    lib = _lib.load()
    Cc = 96
    d = _desc(40, 48, 13, 0)
    planes, _ = _wide_inputs(d, Cc, seed=13)
    rows = d.H * d.W * d.Z
    f = dp.preactivation(*[p.double() for p in planes], (d.H, d.W, d.Z), 0, d.H).reshape(rows, Cc)
    a0 = torch.full((rows, Cc), NAN, device=dev)
    _lib.check(lib.so_tpv_decode_bwd_features(*[ops._p(p) for p in planes], Cc, C.byref(d), 0, d.H, ops._p(a0), ops._stream()), 'features')
    _assert_buckets('a0 = softplus(f), so_tpv_decode_bwd_features', dp.bucket_errors(a0, torch.nn.functional.softplus(f), f))
    sg = torch.ones(rows, Cc, device=dev)
    _lib.check(lib.so_tpv_decode_bwd_input(ops._p(sg), ops._p(a0), sg.numel(), ops._stream()), 'input')
    _assert_buckets('sigmoid(f) from a0, so_tpv_decode_bwd_input', dp.bucket_errors(sg, torch.sigmoid(f), f))
    # hidden: z1 in, a1 = softplus(z1) and g1 = (W2^T g_out) sigmoid(z1) out; with w2 = 1 and g_vol_sdf = 1, g1 = sigmoid(z1)
    z = torch.linspace(-45.0, 45.0, rows * Cc, device=dev).reshape(rows, Cc).contiguous()
    z[0, :8] = torch.tensor([0.0, -0.0, 20.0, -20.0, 1e-39, -1e-39, 16.0, -16.0], device=dev)
    z64 = z.double()
    a1, g1, go = z.clone(), torch.full((rows, Cc), NAN, device=dev), torch.full((rows, 1), NAN, device=dev)
    w2, gvs = torch.ones(1, Cc, device=dev), torch.ones(d.H, d.W, d.zpitch, device=dev)
    gvs[..., d.Z:] = NAN
    _lib.check(lib.so_tpv_decode_bwd_hidden(ops._p(a1), ops._p(gvs), None, ops._p(w2), Cc, C.byref(d), 0, d.H, ops._p(g1), ops._p(go),
                                            ops._stream()), 'hidden')
    assert (go == 1).all()
    _assert_buckets('a1 = softplus(z), so_tpv_decode_bwd_hidden', dp.bucket_errors(a1, torch.nn.functional.softplus(z64), z64))
    _assert_buckets('sigmoid(z), so_tpv_decode_bwd_hidden', dp.bucket_errors(g1, torch.sigmoid(z64), z64))


# ---- 4. backward --------------------------------------------------------------------------------------------------------------
# channels / hidden units moved far negative: (index, shift)
SHIFT_PLANE = ((3, -8.0), (17, -12.0), (40, -8.0), (77, -12.0))
SHIFT_B1 = ((5, -8.0), (50, -8.0), (20, -12.0), (90, -12.0))
# Bars: each error is relative to the max-abs of the reference gradient it is taken over, the whole tensor or one slice of
# it.  d/d b1[j] is a signed sum over all voxels that cancels, so an entry is compared relative to the summed magnitude of
# its terms (b1_mass of the oracle), not to itself.  Measured maxima over every case of this file, native path, on one
# H100 80GB HBM3 at 700 W: per tensor 2.3e-6, per slice 5.1e-6 (b1 entries 7.5e-7).
BAR_TENSOR = 1e-5
BAR_SLICE = 2e-5


def _cotangent(d, kind, seed):
    """(g_vs [H, W, zpitch], g_vf [H, W, Z, feat_pitch] | None) as TPVDecodeFunction.backward receives them, and the oracle's
    [H, W, Z, n_out] view.  'dense': every voxel (sparsity / occupancy lattice losses); 'render': 3 % of the voxels (what rays
    scatter); 'sdf_only' / 'feat_only': the other output took no part in the loss.  The sdf pads carry NaN and the feature
    pad channels 1e30: neither may reach a result."""
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    n_out = 1 + d.n_feat
    go = torch.randn(d.H, d.W, d.Z, n_out, generator=g, device=dev)
    if kind == 'render':
        go *= (torch.rand(d.H, d.W, d.Z, 1, generator=g, device=dev) < 0.03)
    if kind == 'sdf_only':
        go[..., 1:] = 0
    if kind == 'feat_only':
        go[..., 0] = 0
    g_vs = torch.full((d.H, d.W, d.zpitch), NAN, device=dev)
    g_vs[..., :d.Z] = go[..., 0]
    g_vf = None
    if d.n_feat:
        g_vf = torch.full((d.H, d.W, d.Z, d.feat_pitch), 1e30, device=dev)
        g_vf[..., :d.n_feat] = go[..., 1:]
    return g_vs, g_vf, go.double()


def _backward(planes, mlp, d, g_vs, g_vf, mode, monkeypatch):
    from selfocc_b200 import ops
    assert ops.TPVDecodeFunction.SLAB_ROWS == 32
    monkeypatch.setenv('SELFOCC_B200_DECODE_BWD', mode)
    ins = [t.clone().requires_grad_(True) for t in (*planes, *mlp)]
    vs, vf = ops.TPVDecodeFunction.apply(*ins, d)
    if d.n_feat:
        return torch.autograd.grad([vs, vf], ins, [g_vs, g_vf])
    return torch.autograd.grad([vs], ins, [g_vs])


def _grad_report(tag, got, ref, b1_mass):
    """{name: error relative to the tensor's max-abs}, {slice kind: worst error relative to the slice's own max-abs}."""
    from oracle import decode_parity as dp
    per_tensor, per_slice = {}, {}
    for name, a, b in zip(dp.GRAD_NAMES, got, ref):
        assert a.shape == b.shape and torch.isfinite(a).all(), '%s: %s is not finite' % (tag, name)
        scale = float(b.abs().max())
        per_tensor[name] = float((a.double() - b).abs().max()) / scale if scale > 0 else float(a.abs().max())
        if name in dp.PLANE_NAMES:
            per_slice[name + ' per channel'] = float(dp.slice_errors(a, b, 1).max())
        elif name == 'w1':
            per_slice['w1 per column'] = float(dp.slice_errors(a, b, 1).max())
            per_slice['w1 per row'] = float(dp.slice_errors(a, b, 0).max())
        elif name == 'b1':
            per_slice['b1 per entry'] = float(((a.double() - b).abs() / b1_mass).max())
    print('  %s\n    per tensor: %s\n    per slice : %s' % (tag, ' '.join('%s %.1e' % kv for kv in per_tensor.items()),
                                                         ' '.join('%s %.1e' % kv for kv in per_slice.items())))
    return per_tensor, per_slice


def _backward_case(d, cases, monkeypatch, modes=('native', 'torch')):
    """cases: (label, shifted inputs?, cotangent kind).  Collects every miss so one run reports all of them."""
    from oracle import decode_parity as dp
    misses = []
    for i, (label, shifted, kind) in enumerate(cases):
        planes, mlp = _inputs(d, 96, seed=21)
        if shifted:
            for c, s in SHIFT_PLANE:
                planes[0][:, c] += s
            for c, s in SHIFT_B1:
                mlp[1][c] += s
        g_vs, g_vf, go = _cotangent(d, kind, seed=30 + i)
        ref, b1_mass = dp.decode_grads_slabwise(*[p.double() for p in planes], (d.H, d.W, d.Z), *[t.double() for t in mlp], go)
        assert all(float(r.abs().max()) > 0 for r in ref[:5]) and float(b1_mass.min()) > 0
        for mode in modes:
            got = _backward(planes, mlp, d, g_vs, g_vf, mode, monkeypatch)
            tag = '%s, %s cotangent, %s' % (label, kind, mode)
            per_tensor, per_slice = _grad_report(tag, got, ref, b1_mass)
            misses += ['%s: %s %.2e' % (tag, k, v) for k, v in per_tensor.items() if v > BAR_TENSOR]
            misses += ['%s: %s %.2e' % (tag, k, v) for k, v in per_slice.items() if v > BAR_SLICE]
            if kind == 'sdf_only' and d.n_feat:
                assert (got[5][1:] == 0).all() and (got[6][1:] == 0).all()
            if kind == 'feat_only':
                assert got[5][0].abs().max() == 0 and got[6][0] == 0
    assert not misses, '\n'.join(misses)


@gpu
@pytest.mark.parametrize('name', ['nuScenes_depth', 'nuScenes_novel_depth', 'nuScenes_occ', 'KITTI_occ'])
def test_backward_at_shipped_geometry_per_tensor_and_per_channel(name, monkeypatch):
    """H = 257 with the shipped slab of 32 rows: eight full slabs and a one-row last slab."""
    d = _shipped_desc(name)
    print('%s: %d x %d x %d, zpitch %d, %d features' % (name, d.H, d.W, d.Z, d.zpitch, d.n_feat))
    _backward_case(d, (('standard inputs', False, 'dense'), ('standard inputs', False, 'render'),
                       ('shifted inputs', True, 'dense')), monkeypatch)


@gpu
@pytest.mark.parametrize('H', [20, 33])
def test_backward_short_slab_and_absent_cotangents(H, monkeypatch):
    """H = 20: one slab shorter than the slab height; H = 33: a full slab and a one-row slab.  One output without a cotangent."""
    d = _desc(H, 19, 6, 3)
    _backward_case(d, (('H %d standard' % H, False, 'dense'), ('H %d standard' % H, False, 'sdf_only'),
                       ('H %d standard' % H, False, 'feat_only'), ('H %d shifted' % H, True, 'render')), monkeypatch)
