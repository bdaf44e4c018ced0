"""Oracle: the voxel-cube picture and the voxel face mesh in numpy / fp64 (test infrastructure).

Restates so_voxel_render / so_voxel_faces_* by different algorithms:
* cameras from VTK's own matrices: the view transform of vtkPerspectiveTransform::SetupCamera, vtkCamera::Elevation as
  Translate(fp) RotateWXYZ(angle, -right) Translate(-fp) on homogeneous points (Rodrigues' formula), OrthogonalizeViewUp as
  the view matrix's second row, and pixel rays by unprojecting NDC points through the inverse of VTK's perspective
  projection times the view transform;
* the picture: for each pixel ray, a slab test against every drawn voxel's cube, keeping the nearest entry within
  [near, far] (ties: the lowest voxel index), its face the axis of the latest slab entry;
* the faces: exposed faces from shifted copies of the drawn mask, sorted by voxel index then face code, corners by the
  quad rule of include/selfocc_b200.h.
Grid: labels [H, W, D], voxel (h, w, d) = cube [origin + (w, h, d) vs, origin + (w + 1, h + 1, d + 1) vs], origin and vs
rounded to fp32 as the kernels receive them.
"""
import math
import numpy as np


# ------------------------------------------------------------------------------------------------------------ cameras
def view_matrix(position, focal_point, view_up):
    """VTK's 4x4 view transform: rows right, ortho up, view-plane normal, then the translation to the camera."""
    p, f, up = (np.asarray(v, dtype=np.float64) for v in (position, focal_point, view_up))
    vpn = (p - f) / np.linalg.norm(p - f)
    side = np.cross(up, vpn)
    side /= np.linalg.norm(side)
    oup = np.cross(vpn, side)
    V = np.eye(4)
    V[0, :3], V[1, :3], V[2, :3] = side, oup, vpn
    V[:3, 3] = -V[:3, :3] @ p
    return V


def _rodrigues(angle_deg, axis):
    k = np.asarray(axis, dtype=np.float64)
    k = k / np.linalg.norm(k)
    a = math.radians(angle_deg)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(a) * Kx + (1 - math.cos(a)) * (Kx @ Kx)


def elevation(position, focal_point, view_up, angle_deg):
    """vtkCamera::Elevation then OrthogonalizeViewUp -> (position, view_up)."""
    V = view_matrix(position, focal_point, view_up)
    axis = -V[0, :3]
    f = np.asarray(focal_point, dtype=np.float64)
    T = np.eye(4)
    T[:3, 3] = f
    R = np.eye(4)
    R[:3, :3] = _rodrigues(angle_deg, axis)
    Tb = np.eye(4)
    Tb[:3, 3] = -f
    pos = (T @ R @ Tb @ np.append(np.asarray(position, dtype=np.float64), 1.0))[:3]
    return pos, view_matrix(pos, focal_point, view_up)[1, :3].copy()


def vis3d_nuscenes_ref():
    """vis_3d.py:311-326 -> (position, focal_point, view_up, view_angle, clip)."""
    pos = np.array([-107.15500034628069, -0.008333206176756742, 92.16667026873841])
    fp = np.array([0.008333206176757812, -0.008333206176757812, 1.399999976158142])
    up = np.array([0.6463156430702277, -6.4549254142909245e-18, 0.7630701733934555])
    for deg in (5, 5, -5):
        pos, up = elevation(pos, fp, up, deg)
    return pos, fp, up, 30.0, (78.84362692774403, 218.2948716014858)


def perspective(view_angle, aspect, near, far):
    """vtkPerspectiveTransform::Perspective (the projection of a vtkCamera with a vertical view angle)."""
    ymax = math.tan(math.radians(view_angle) / 2.0) * near
    xmax = ymax * aspect
    P = np.zeros((4, 4))
    P[0, 0] = near / xmax
    P[1, 1] = near / ymax
    P[2, 2] = -(far + near) / (far - near)
    P[2, 3] = -2.0 * far * near / (far - near)
    P[3, 2] = -1.0
    return P


def camera_rays(position, focal_point, view_up, view_angle, image_size, clip):
    """Per-pixel rays of a VTK camera by unprojection -> origin [3], directions [h, w, 3] scaled to unit depth along the
    view direction (so the ray parameter is the depth the clipping range bounds)."""
    h, w = image_size
    near, far = clip
    PV = perspective(view_angle, w / h, near, far) @ view_matrix(position, focal_point, view_up)
    inv = np.linalg.inv(PV)
    u, v = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    x, y = 2.0 * u / w - 1.0, 1.0 - 2.0 * v / h
    pts = []
    for z in (-1.0, 1.0):
        q = np.stack([x, y, np.full_like(x, z), np.ones_like(x)], -1) @ inv.T
        pts.append(q[..., :3] / q[..., 3:])
    d = pts[1] - pts[0]
    fwd = np.asarray(focal_point, dtype=np.float64) - np.asarray(position, dtype=np.float64)
    fwd /= np.linalg.norm(fwd)
    d = d / (d @ fwd)[..., None]
    return np.asarray(position, dtype=np.float64), d


def rays_from_rows(rows, image_size):
    """so_voxel_render's camera rows [K, 16] (fp32 values) -> origins [K, 3], directions [K, h, w, 3], near [K], far [K]
    in fp64."""
    r = np.asarray(rows, dtype=np.float64).reshape(-1, 16)
    h, w = image_size
    u, v = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    pix = np.stack([u, v, np.ones_like(u)], -1)
    M = r[:, 3:12].reshape(-1, 3, 3)
    d = np.einsum('kij,hwj->khwi', M, pix)
    return r[:, :3], d, r[:, 12], r[:, 13]


# ------------------------------------------------------------------------------------------------------------ picture
def grid32(origin, vs):
    """The grid as so_voxel_render receives it: origin and voxel size rounded to fp32, then held in fp64."""
    return np.asarray(origin, dtype=np.float32).astype(np.float64), float(np.float32(vs))


def _boxes(shape, origin, vs, idx):
    H, W, D = shape
    hh, ww, dd = idx // (W * D), (idx // D) % W, idx % D
    cell = np.stack([ww, hh, dd], -1).astype(np.float64)
    org, vs = grid32(origin, vs)
    return org + cell * vs, org + (cell + 1.0) * vs


def slab(o, d, lo, hi):
    """Ray o + t d against boxes [lo, hi] -> (t_in, t_out, entry axis) over broadcast shapes; a zero direction component
    keeps the ray inside that slab when lo <= o <= hi, else outside."""
    with np.errstate(divide='ignore', invalid='ignore'):
        t1 = (lo - o) / d
        t2 = (hi - o) / d
    zero = d == 0
    inside = (lo <= o) & (o <= hi)
    tl = np.where(zero, np.where(inside, -np.inf, np.inf), np.minimum(t1, t2))
    th = np.where(zero, np.where(inside, np.inf, -np.inf), np.maximum(t1, t2))
    return tl.max(-1), th.min(-1), tl.argmax(-1)


def _exposed26(drawn_v):
    """Drawn voxels with a non-drawn or outside 26-neighbour."""
    p = np.pad(drawn_v, 1)
    H, W, D = drawn_v.shape
    allin = np.ones_like(drawn_v)
    for a in (0, 1, 2):
        for b in (0, 1, 2):
            for c in (0, 1, 2):
                allin &= p[a:a + H, b:b + W, c:c + D]
    return drawn_v & ~allin


def render_ref(labels, origin, vs, o, d, near, far, drawn, budget=1 << 20):
    """Nearest drawn voxel entered within [near, far] for rays o [3] + t d [P, 3] from one camera -> (voxel int64 [P] or
    -1, face int64 [P] or -1, t_in fp64 [P] or inf); equal entries go to the lowest voxel index.  Only voxels with an
    undrawn 26-neighbour can be entered first from undrawn space; a ray whose point at near lies within 1e-9 of a drawn
    voxel is tested against every drawn voxel."""
    labels = np.asarray(labels)
    drawn_v = np.asarray(drawn, dtype=bool)[labels]
    shape = labels.shape
    d = np.asarray(d, dtype=np.float64).reshape(-1, 3)
    o = np.broadcast_to(np.asarray(o, dtype=np.float64), d.shape)
    P = d.shape[0]
    full = np.flatnonzero(drawn_v)
    cull = np.flatnonzero(_exposed26(drawn_v))
    # rays starting (at near) in or at a drawn voxel
    p0 = o + near * d
    start_in = np.zeros(P, dtype=bool)
    org, vs32 = grid32(origin, vs)
    H, W, D = shape
    n = np.array([W, H, D])
    for corner in range(8):
        off = np.array([(corner >> k) & 1 for k in range(3)]) * 2e-9 - 1e-9
        c = np.floor((p0 + off - org) / vs32).astype(np.int64)
        ok = ((c >= 0) & (c < n)).all(-1)
        cc = np.where(ok[:, None], c, 0)
        start_in |= ok & drawn_v[cc[:, 1], cc[:, 0], cc[:, 2]]
    vox = np.full(P, -1, dtype=np.int64)
    face = np.full(P, -1, dtype=np.int64)
    tin = np.full(P, np.inf)
    dn = np.linalg.norm(d, axis=-1)
    for rays, cand in ((np.flatnonzero(~start_in), cull), (np.flatnonzero(start_in), full)):
        if rays.size == 0 or cand.size == 0:
            continue
        # candidates by the distance of their centre from the camera: a cube whose centre lies r away is entered no nearer
        # than r - (sqrt(3) / 2) vs, so a ray whose best entry is nearer than that for every remaining cube is settled
        lo, hi = _boxes(shape, origin, vs, cand)
        r = np.linalg.norm((lo + hi) / 2 - o[rays[0]], axis=-1)
        order = np.argsort(r, kind='stable')
        lo, hi, cand, r = lo[order], hi[order], cand[order], r[order]
        active, s = rays, 0
        while s < cand.size and active.size:
            e = min(cand.size, s + max(1024, budget // active.size))
            tl, th, ax = slab(o[active, None, :], d[active, None, :], lo[None, s:e], hi[None, s:e])
            tt = np.where((tl <= th) & (tl >= near) & (tl <= far), tl, np.inf)
            bt = tt.min(1)
            j = np.argmin(np.where(tt == bt[:, None], cand[None, s:e], np.iinfo(np.int64).max), 1)   # lowest index
            ar = np.arange(active.size)
            bi = cand[s + j]
            better = np.isfinite(bt) & ((bt < tin[active]) | ((bt == tin[active]) & (bi < vox[active])))
            upd = active[better]
            a = ax[ar, j][better]
            vox[upd], tin[upd], face[upd] = bi[better], bt[better], 2 * a + (d[upd, a] < 0)
            s = e
            if s < cand.size:
                active = active[~(tin[active] * dn[active] < r[s] - 0.87 * vs32)]
    return vox, face, tin


def voxel_entry(labels_shape, origin, vs, o, d, idx):
    """Slab entry / exit of the given voxels for rays o + t d [P, 3] -> (t_in, t_out, per-axis entries [P, 3])."""
    lo, hi = _boxes(labels_shape, origin, vs, np.maximum(np.asarray(idx), 0))
    d = np.asarray(d, dtype=np.float64).reshape(-1, 3)
    o = np.broadcast_to(np.asarray(o, dtype=np.float64), d.shape)
    with np.errstate(divide='ignore', invalid='ignore'):
        t1, t2 = (lo - o) / d, (hi - o) / d
    inside = (lo <= o) & (o <= hi)
    tl = np.where(d == 0, np.where(inside, -np.inf, np.inf), np.minimum(t1, t2))
    th = np.where(d == 0, np.where(inside, np.inf, -np.inf), np.maximum(t1, t2))
    return tl.max(-1), th.min(-1), tl


def ties(labels, origin, vs, o, d, near, far, vox_a, face_a, vox_b, face_b, t_b, tol_vox=1e-4):
    """Pixels where answer a (voxel, face) and answer b (voxel, face, fp64 entry t_b) differ only by a tie: the fp64
    entries of the two candidate voxels, or of a candidate and a clip plane or its own exit, lie within tol_vox voxel of
    each other along the ray; for the same voxel, two of its slab entries do."""
    shape = labels.shape
    dn = np.linalg.norm(d, axis=-1)
    tol = tol_vox * vs / dn
    ta, tao, ax_a = voxel_entry(shape, origin, vs, o, d, vox_a)
    ta = np.where(vox_a >= 0, ta, np.inf)
    tb = np.where(vox_b >= 0, t_b, np.inf)
    same = vox_a == vox_b
    with np.errstate(invalid='ignore'):                      # inf - inf where neither side hits: not a tie
        face_tie = same & (np.abs(np.sort(ax_a, -1)[:, -1] - np.sort(ax_a, -1)[:, -2]) < tol)
        vox_tie = ~same & (np.abs(ta - tb) < tol)
        clip_tie = ~same & ((np.abs(np.minimum(ta, tb) - near) < tol) | (np.abs(np.minimum(ta, tb) - far) < tol)
                            | (np.abs(tao - ta) < tol))
    return face_tie | vox_tie | clip_tie


def shade_rgb(labels, vox, face, palette, shade, background):
    """The colour rule in fp32: round-half-even(palette[label].rgb * shade[face]), background without a hit."""
    lab = np.asarray(labels).reshape(-1)[np.maximum(vox, 0)]
    pal = np.asarray(palette, dtype=np.float32)[lab, :3]
    s = np.asarray(shade, dtype=np.float32)[np.maximum(face, 0)]
    rgb = np.clip(np.rint(pal * s[:, None]), 0, 255).astype(np.uint8)
    rgb[vox < 0] = np.asarray(background, dtype=np.uint8)
    return rgb


# ------------------------------------------------------------------------------------------------------------ faces
def faces_ref(labels, origin, vs, drawn):
    """Exposed faces of the drawn voxels -> {'vertices' fp32 [4F, 3], 'faces' int64 [2F, 3], 'normals' fp32 [4F, 3],
    'sem' uint8 [4F]} in ascending voxel index then face code."""
    labels = np.asarray(labels)
    dv = np.asarray(drawn, dtype=bool)[labels]
    H, W, D = dv.shape
    p = np.pad(dv, 1)
    # neighbour across face 2a + s: array axis of x is 1 (w), of y 0 (h), of z 2 (d)
    exposed = np.zeros((H, W, D, 6), dtype=bool)
    for f in range(6):
        a, s = f >> 1, 1 if f & 1 else -1
        sl = [slice(1, H + 1), slice(1, W + 1), slice(1, D + 1)]
        arr_axis = (1, 0, 2)[a]
        sl[arr_axis] = slice(1 + s, (H, W, D)[arr_axis] + 1 + s)
        exposed[..., f] = dv & ~p[tuple(sl)]
    idx, f = np.nonzero(exposed.reshape(-1, 6))
    hh, ww, dd = idx // (W * D), (idx // D) % W, idx % D
    cell = np.stack([ww, hh, dd], -1)
    a, up = f >> 1, f & 1
    b, c = (a + 1) % 3, (a + 2) % 3
    cb = np.array([[0, 0, 1, 1], [0, 1, 1, 0]])[up]       # lower face: (0,0) (0,1) (1,1) (1,0); upper: (0,0) (1,0) (1,1) (0,1)
    cc = np.array([[0, 1, 1, 0], [0, 0, 1, 1]])[up]
    F = idx.size
    corner = np.repeat(cell[:, None, :], 4, 1)
    ar = np.arange(F)
    for k in range(4):
        corner[ar, k, a] += up
        corner[ar, k, b] += cb[:, k]
        corner[ar, k, c] += cc[:, k]
    org = np.float32(origin).astype(np.float64)
    vertices = (org + corner.astype(np.float64) * np.float64(np.float32(vs))).astype(np.float32).reshape(-1, 3)
    normals = np.zeros((F, 4, 3), dtype=np.float32)
    normals[ar, :, a] = np.where(up, 1.0, -1.0)[:, None]
    v0 = 4 * np.arange(F)[:, None]
    faces = np.concatenate([v0 + np.array([0, 1, 2]), v0 + np.array([0, 2, 3])], 1).reshape(-1, 3)
    sem = np.repeat(labels.reshape(-1)[idx], 4).astype(np.uint8)
    return dict(vertices=vertices, faces=faces, normals=normals.reshape(-1, 3), sem=sem)
