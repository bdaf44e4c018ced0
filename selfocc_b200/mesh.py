"""The scene surface straight from the decoded volume: marching cubes over the lattice of ``NeuSHead.get_uniform_sdf``.

The reference's 3D visualisation (vis_3d.py, vis_3d_scene.py) builds ``forward_occ``'s whole lattice, copies it to the
host and draws voxel glyphs.  Here two kernels (so_mesh_count / so_mesh_emit) evaluate the field at the lattice points on
the fly and write only the mesh.  A point is inside when ``sdf <= thresh``, the rule of eval_iou.py and
``NeuSHead.occupancy``, so the surface bounds exactly the points that ``occupancy`` labels occupied.  Per-vertex
attributes come from the field query at the vertices.
"""
import ctypes as C
import numpy as np
import torch

from . import _lib
from .occupancy import as_lut
from .ops import _chk, _p, _stream, field_query

SH_C0 = 0.28209479177387814          # sh_render.py:4, the render's kC0
ATTR_CHUNK = 1 << 20                 # vertices per field query in vertex_attributes: bounds its scratch


def marching_cubes(vol_sdf, desc, axes, thresh=0.0):
    """Mesh of the level set ``sdf = thresh`` on the lattice ``axes`` = (xs [nx], ys [ny], zs [nz]) (layout [ny, nx, nz])
    -> (vertices fp32 [V, 3] lidar-frame metres, faces int32 [F, 3]).  Faces run counter-clockwise seen from the outside
    (sdf > thresh).  One synchronising read (the two totals); an empty surface launches no emit pass."""
    lib = _lib.load()
    xs, ys, zs = (a.contiguous() for a in axes)
    _chk(vol_sdf, name='vol_sdf')
    for a, name in ((xs, 'xs'), (ys, 'ys'), (zs, 'zs')):
        _chk(a, name=name)
    dev = vol_sdf.device
    lattice = (_p(xs), len(xs), _p(ys), len(ys), _p(zs), len(zs))
    n = len(xs) * len(ys) * len(zs)
    counts = torch.empty(2, n, dtype=torch.int32, device=dev)
    edge_mask = torch.empty(n, dtype=torch.uint8, device=dev)
    _lib.check(lib.so_mesh_count(_p(vol_sdf), C.byref(desc), *lattice, float(thresh), _p(counts), _p(edge_mask), _stream()),
               'so_mesh_count')
    # one 1-D scan per row: ATen hands a 1-D scan to its device-wide scan, while a scan along the last dimension of the
    # [2, N] tensor would run with one CTA per row
    scans = torch.empty_like(counts)
    for row in range(2):
        torch.cumsum(counts[row], 0, dtype=torch.int32, out=scans[row])
    n_vertices, n_faces = counts.sum(1, dtype=torch.int64).tolist()        # the one host read
    if n_vertices >= 2 ** 31 or n_faces >= 2 ** 31:
        raise _lib.SelfOccLibraryError('marching_cubes: %d vertices, %d faces: ids need more than int32' % (n_vertices, n_faces))
    vertices = torch.empty(n_vertices, 3, device=dev)
    faces = torch.empty(n_faces, 3, dtype=torch.int32, device=dev)
    if n_vertices:
        _lib.check(lib.so_mesh_emit(_p(vol_sdf), C.byref(desc), *lattice, float(thresh), _p(scans), _p(edge_mask), n_vertices,
                                    n_faces, _p(vertices), _p(faces), _stream()), 'so_mesh_emit')
    return vertices, faces


def vertex_attributes(vol_sdf, vol_feat, desc, vertices, n_sem=0, lut=None, rgb=False, sh_act='relu', chunk=ATTR_CHUNK):
    """Field attributes at ``vertices`` [V, 3], from the field query in chunks of ``chunk`` vertices:
    'normals' fp32 [V, 3], the normalised sdf gradient; 'sem' uint8 [V] (n_sem > 0), lut[argmax] of feature channels
    3 .. 3 + n_sem (first maximum; lut None: the raw argmax); 'rgb' fp32 [V, 3] (rgb), the view-independent SH degree-0
    colour of channels 0 .. 2 under the render's ``sh_act`` ('relu': relu(C0 f + 1/2), 'sigmoid': sigmoid(C0 f))."""
    dev = vertices.device
    V = vertices.shape[0]
    lut = as_lut(lut, dev) if n_sem else None
    if lut is not None and lut.numel() != n_sem:
        raise ValueError('lut has %d entries, the head has %d semantic channels' % (lut.numel(), n_sem))
    if sh_act not in ('relu', 'sigmoid'):
        raise ValueError('sh_act must be relu or sigmoid, got %r' % (sh_act,))
    out = {'normals': torch.empty(V, 3, device=dev)}
    if n_sem:
        out['sem'] = torch.empty(V, dtype=torch.uint8, device=dev)
    if rgb:
        out['rgb'] = torch.empty(V, 3, device=dev)
    for b in range(0, V, chunk):
        e = min(V, b + chunk)
        _, grad, feat = field_query(vol_sdf, vol_feat, desc, vertices[b:e].contiguous(), want_grad=True, want_feat=bool(n_sem or rgb))
        out['normals'][b:e] = torch.nn.functional.normalize(grad, dim=-1)
        if n_sem:
            arg = torch.argmax(feat[:, 3:3 + n_sem], dim=-1)
            out['sem'][b:e] = lut[arg] if lut is not None else arg.to(torch.uint8)
        if rgb:
            raw = feat[:, :3] * SH_C0
            out['rgb'][b:e] = (raw + 0.5).clamp_min(0.0) if sh_act == 'relu' else torch.sigmoid(raw)
    return out


def _palette(n):
    """A fixed colour per label for meshes with labels and no colour map."""
    return np.random.default_rng(0).integers(48, 256, size=(max(n, 1), 3), dtype=np.uint8)


def write_ply(path, mesh, colormap=None):
    """Write ``mesh`` (NeuSHead.mesh's dict: 'vertices', 'faces', 'normals', optional 'sem' / 'rgb') as a binary
    little-endian PLY with per-vertex position, normal and colour.  Colour: ``colormap`` [n_labels, 3 or 4] (RGB or RGBA;
    integers are 0..255, floats 0..1; alpha is dropped) indexed by 'sem' when given, else 'rgb', else 'sem' through a
    fixed palette; no colour without either."""
    v = mesh['vertices'].detach().cpu().numpy().astype('<f4')
    f = mesh['faces'].detach().cpu().numpy().astype('<i4')
    nrm = mesh['normals'].detach().cpu().numpy().astype('<f4')
    sem = mesh['sem'].detach().cpu().numpy() if 'sem' in mesh else None
    col = None
    if colormap is not None:
        if sem is None:
            raise ValueError('a colormap needs per-vertex labels (a return_sem head)')
        cm = np.asarray(colormap)[:, :3]
        cm = np.clip(np.rint(cm * 255.0) if np.issubdtype(cm.dtype, np.floating) else cm, 0, 255).astype(np.uint8)
        col = cm[sem]
    elif 'rgb' in mesh:
        col = np.clip(np.rint(mesh['rgb'].detach().cpu().numpy() * 255.0), 0, 255).astype(np.uint8)
    elif sem is not None:
        col = _palette(int(sem.max()) + 1 if sem.size else 1)[sem]
    vtype = [('x', '<f4'), ('y', '<f4'), ('z', '<f4'), ('nx', '<f4'), ('ny', '<f4'), ('nz', '<f4')]
    if col is not None:
        vtype += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1')]
    va = np.empty(len(v), dtype=vtype)
    for i, k in enumerate(('x', 'y', 'z')):
        va[k] = v[:, i]
        va['n' + k] = nrm[:, i]
    if col is not None:
        for i, k in enumerate(('red', 'green', 'blue')):
            va[k] = col[:, i]
    fa = np.empty(len(f), dtype=[('n', 'u1'), ('v', '<i4', (3,))])
    fa['n'] = 3
    fa['v'] = f
    props = ''.join('property %s %s\n' % ('float' if t == '<f4' else 'uchar', k) for k, t in vtype)
    head = ('ply\nformat binary_little_endian 1.0\nelement vertex %d\n%selement face %d\n'
            'property list uchar int vertex_indices\nend_header\n' % (len(v), props, len(f)))
    with open(path, 'wb') as fh:
        fh.write(head.encode('ascii'))
        fh.write(va.tobytes())
        fh.write(fa.tobytes())
