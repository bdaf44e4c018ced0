"""The label volume drawn as voxel cubes on the device: the picture vis_3d.py / vis_3d_scene.py make with mayavi.

The reference copies ``forward_occ``'s lattice to the host and has mayavi draw every occupied voxel as a cube glyph
(``mlab.points3d(..., mode='cube')``) from fixed VTK cameras into 2560 x 1440 PNGs.  Here ``NeuSHead.occupancy`` gives the
same label volume on the device, and one kernel (so_voxel_render) ray-casts it for K cameras at once:

* grid: labels uint8 [H, W, D] in the layout ``NeuSHead.occupancy`` returns; voxel [h, w, d] is the cube of side
  ``voxel_size`` centred at ``origin + (w + 1/2, h + 1/2, d + 1/2) * voxel_size``, which is where vis_3d.py's
  ``get_grid_coords`` (``np.meshgrid``'s default 'xy' indexing) and its flattening of the volume put it on a square grid:
  the first array axis runs along y;
* a label is drawn when the palette gives it a non-zero alpha (the vis_3d palettes below: ``0 < label < 100``);
* a pixel shows the first drawn voxel its ray enters within the camera's [near, far], coloured
  ``round(palette[label].rgb * shade[face])`` by the face it entered through; no hit shows the background.

``voxel_mesh`` writes the same cubes' exposed faces as a mesh (so_voxel_faces_count / so_voxel_faces_emit) that
``mesh.write_ply`` writes unchanged.  Cameras follow VTK's semantics (``look_at``, ``elevate``); the presets restate
vis_3d.py's camera calls.
"""
import ctypes as C
import math
import struct
import zlib

import numpy as np
import torch

from . import _lib
from .ops import _p, _stream

# Shade per face code 2a + s (axis a: 0 x, 1 y, 2 z; s = 0 the cube's lower face on that axis, 1 its upper face): the
# upper z face (seen from above) is full brightness, x faces 0.8, y faces 0.65, the lower z face 0.5.  A fixed-light
# stand-in for VTK's headlight shading of the glyph faces.
SHADE = (0.8, 0.8, 0.65, 0.65, 0.5, 1.0)
BACKGROUND = (255, 255, 255)               # mlab.figure(bgcolor=(1, 1, 1))
IMAGE_SIZE = (1440, 2560)                  # (height, width): mlab.figure(size=(2560, 1440))
FACE_NAMES = ('-x', '+x', '-y', '+y', '-z', '+z')

# vis_3d.py:186-206, the nuScenes table drawn with vmin=1, vmax=16 (labels through OPENSEED2NUSCENES)
NUSCENES_COLORS = (
    (255, 120, 50, 255), (255, 192, 203, 255), (255, 255, 0, 255), (0, 150, 245, 255), (0, 255, 255, 255),
    (255, 127, 0, 255), (255, 0, 0, 255), (255, 240, 150, 255), (135, 60, 0, 255), (160, 32, 240, 255),
    (255, 0, 255, 255), (139, 137, 137, 255), (75, 0, 75, 255), (150, 240, 80, 255), (230, 230, 250, 255),
    (0, 175, 0, 255))
# vis_pics.py create_label_colormap (the Cityscapes colours), drawn for KITTI with vmin=1, vmax=19 and alpha 255
KITTI_COLORS = (
    (128, 64, 128), (244, 35, 232), (70, 70, 70), (102, 102, 156), (190, 153, 153), (153, 153, 153), (250, 170, 30),
    (220, 220, 0), (107, 142, 35), (152, 251, 152), (70, 130, 180), (220, 20, 60), (255, 0, 0), (0, 0, 142), (0, 0, 70),
    (0, 60, 100), (0, 80, 100), (0, 0, 230), (119, 11, 32))

DRAWN_MAX = 100                            # vis_3d.py:143-145: labels in (0, 100) are drawn


def _drawn_labels():
    l = np.arange(256)
    return (l > 0) & (l < DRAWN_MAX)


def table_palette(colors):
    """RGBA [256, 4] uint8 of a glyph table drawn with vmin=1, vmax=len(colors): VTK's lookup maps label l to row
    floor((l - 1) n / (n - 1)) clamped to [0, n - 1], which is row l - 1 for 1 <= l <= n and the last row above; labels
    outside (0, 100) get alpha 0."""
    c = np.asarray(colors, dtype=np.uint8)
    if c.shape[1] == 3:
        c = np.concatenate([c, np.full((len(c), 1), 255, np.uint8)], 1)
    l = np.arange(256)
    pal = c[np.clip(l - 1, 0, len(c) - 1)].copy()
    pal[~_drawn_labels(), 3] = 0
    return pal


NUSCENES_PALETTE = table_palette(NUSCENES_COLORS)
KITTI_PALETTE = table_palette(KITTI_COLORS)


def jet(vmin, vmax):
    """RGBA [256, 4] uint8 for vis_3d.py's non-semantic branch (``colormap='jet'``, scalar range [vmin, vmax], mayavi's
    default: the data's range).  Label l takes entry i = clamp(floor((l - vmin) / (vmax - vmin) * 256), 0, 255) of a
    256-entry table, as VTK's lookup does; the table is the standard analytic jet, r, g, b = clip(1.5 - |4x - 3|,
    1.5 - |4x - 2|, 1.5 - |4x - 1|) at x = i / 255, which approximates VTK's jet table rather than reproducing it.
    Labels outside (0, 100) get alpha 0."""
    l = np.arange(256, dtype=np.float64)
    span = max(float(vmax) - float(vmin), 1e-12)
    i = np.clip(np.floor((l - vmin) / span * 256.0), 0, 255)
    x = i / 255.0
    rgb = np.clip(np.stack([1.5 - np.abs(4 * x - 3), 1.5 - np.abs(4 * x - 2), 1.5 - np.abs(4 * x - 1)], -1), 0.0, 1.0)
    pal = np.empty((256, 4), np.uint8)
    pal[:, :3] = np.rint(rgb * 255.0)
    pal[:, 3] = np.where(_drawn_labels(), 255, 0)
    return pal


def height_labels(occ, cap=0):
    """vis_3d.py:585,609-611: occupied voxels of [H, W, D] labelled z + 1 by their layer z, the top ``cap`` layers
    cleared -> uint8 [H, W, D] on occ's device (draw with ``jet(1, D - cap)``)."""
    D = occ.shape[-1]
    z = torch.arange(1, D + 1, device=occ.device, dtype=torch.uint8)
    keep = (occ != 0) & (z <= D - cap)
    return torch.where(keep, z, torch.zeros((), dtype=torch.uint8, device=occ.device))


# ---------------------------------------------------------------------------------------------------------------------
# cameras


class Camera:
    """A VTK-style perspective camera in fp64: position, focal point, view-up, vertical view angle (degrees), image size
    (height, width) and clipping range (near, far) along the view direction."""

    def __init__(self, position, focal_point, view_up, view_angle, image_size, clip):
        self.position = np.asarray(position, dtype=np.float64).copy()
        self.focal_point = np.asarray(focal_point, dtype=np.float64).copy()
        self.view_up = np.asarray(view_up, dtype=np.float64).copy()
        self.view_angle = float(view_angle)
        self.image_size = (int(image_size[0]), int(image_size[1]))
        self.clip = (float(clip[0]), float(clip[1]))

    def frame(self):
        """(right, ortho view-up, view-plane normal): the rows of VTK's view rotation (vtkPerspectiveTransform::
        SetupCamera): vpn = |position - focal|, right = |view_up x vpn|, up = vpn x right."""
        vpn = self.position - self.focal_point
        vpn = vpn / np.linalg.norm(vpn)
        right = np.cross(self.view_up, vpn)
        right = right / np.linalg.norm(right)
        return right, np.cross(vpn, right), vpn

    def row(self):
        """The 16 floats so_voxel_render reads: origin, the row-major 3x3 matrix taking a pixel centre (u + 1/2, v + 1/2,
        1) to its ray direction, near, far, 0, 0.  The direction has a unit component along the view axis, so the ray
        parameter is the depth that the clipping range bounds."""
        right, up, vpn = self.frame()
        h, w = self.image_size
        f = 0.5 * h / math.tan(math.radians(self.view_angle) / 2.0)
        M = np.stack([right / f, -up / f, -vpn - (0.5 * w / f) * right + (0.5 * h / f) * up], 1)
        return np.concatenate([self.position, M.reshape(-1), self.clip, (0.0, 0.0)])

    def resized(self, image_size):
        """The same view at another image size (the view angle stays vertical)."""
        return Camera(self.position, self.focal_point, self.view_up, self.view_angle, image_size, self.clip)


def look_at(position, focal_point, view_up=(0.0, 0.0, 1.0), view_angle=30.0, image_size=IMAGE_SIZE, clip=(0.01, 300.0)):
    """A camera set as vis_3d.py sets mayavi's: position, focal point, view-up, vertical view angle in degrees."""
    return Camera(position, focal_point, view_up, view_angle, image_size, clip)


def _rotate_wxyz(angle_deg, axis):
    """vtkTransform::RotateWXYZ: rotation by angle (degrees, right hand) about axis, from the unit quaternion."""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    h = math.radians(angle_deg) / 2.0
    w, (x, y, z) = math.cos(h), a * math.sin(h)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def elevate(cam, degrees):
    """vtkCamera::Elevation(degrees) then OrthogonalizeViewUp: rotate the position about the focal point around minus
    the view's right axis, then set the view-up to the new view's orthogonal up."""
    right, _, _ = cam.frame()
    R = _rotate_wxyz(degrees, -right)
    out = Camera(cam.focal_point + R @ (cam.position - cam.focal_point), cam.focal_point, cam.view_up, cam.view_angle,
                 cam.image_size, cam.clip)
    out.view_up = out.frame()[1]
    return out


def _vis3d_nuscenes():
    """vis_3d.py:304-326: the last camera set explicitly, then Elevation(5), Elevation(5), Elevation(-5), each followed
    by OrthogonalizeViewUp; the clipping range stays the one set last."""
    cam = look_at([-107.15500034628069, -0.008333206176756742, 92.16667026873841],
                  [0.008333206176757812, -0.008333206176757812, 1.399999976158142],
                  [0.6463156430702277, -6.4549254142909245e-18, 0.7630701733934555], 30.0, IMAGE_SIZE,
                  (78.84362692774403, 218.2948716014858))
    for deg in (5, 5, -5):
        cam = elevate(cam, deg)
    return cam


VIS3D_NUSCENES = _vis3d_nuscenes()


def kitti_camera(metas, image_size=IMAGE_SIZE):
    """vis_3d.py:328-335, the KITTI branch: the frame's ``cam_positions[0]`` / ``focal_positions[0]``, view-up z,
    view angle 41, clipping range [0.01, 300]."""
    return look_at(metas['cam_positions'][0], metas['focal_positions'][0], (0.0, 0.0, 1.0), 41.0, image_size, (0.01, 300.0))


def from_img2lidar(M, image_size, out_size=None, clip=(0.01, 300.0)):
    """The frame's own cameras in the head's Img2LiDAR convention: M [N, 4, 4] (tensor or array) maps (x d, y d, d, 1),
    (x, y) image coordinates of an ``image_size`` = (height, width) image, to lidar metres.  -> camera rows [N, 16] fp32
    (a tensor on M's device, built there without a host read) for rendering at ``out_size`` (default image_size): pixel
    centre (u + 1/2, v + 1/2) of the output is image point ((u + 1/2) W / w, (v + 1/2) H / h), its ray parameter is
    the camera depth and ``clip`` bounds it."""
    M = torch.as_tensor(M)
    M = M.reshape(-1, 4, 4).to(torch.float64)
    h, w = out_size if out_size is not None else image_size
    R = M[:, :3, :3].clone()
    R[:, :, 0] *= image_size[1] / w
    R[:, :, 1] *= image_size[0] / h
    tail = torch.zeros(M.shape[0], 4, dtype=M.dtype, device=M.device)
    tail[:, 0], tail[:, 1] = clip[0], clip[1]
    return torch.cat([M[:, :3, 3], R.reshape(-1, 9), tail], 1).to(torch.float32).contiguous()


def camera_rows(cameras, device):
    """Cameras (a Camera, a list of Cameras, or rows [K, 16] as an array or tensor) -> contiguous, 16-byte aligned fp32
    [K, 16] on ``device``.  Host rows go up from pinned memory without blocking."""
    if isinstance(cameras, Camera):
        cameras = [cameras]
    if isinstance(cameras, (list, tuple)) and cameras and isinstance(cameras[0], Camera):
        cameras = np.stack([c.row() for c in cameras])
    if torch.is_tensor(cameras) and cameras.is_cuda:
        rows = cameras.to(device=device, dtype=torch.float32)
    else:
        host = torch.as_tensor(np.asarray(cameras, dtype=np.float32) if not torch.is_tensor(cameras) else cameras,
                               dtype=torch.float32)
        rows = host.contiguous().pin_memory().to(device, non_blocking=True)
    rows = rows.reshape(-1, 16).contiguous()
    if rows.data_ptr() % 16:
        rows = rows.clone()
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# device passes


def _grid(labels, origin):
    if not (torch.is_tensor(labels) and labels.is_cuda):
        raise RuntimeError('voxel_vis: labels must be a CUDA tensor (there is no CPU fallback)')
    if labels.dtype != torch.uint8 or labels.dim() != 3:
        raise ValueError('labels must be uint8 [H, W, D], got %s %s' % (labels.dtype, tuple(labels.shape)))
    o = (C.c_float * 3)(*[float(v) for v in origin])
    return labels.contiguous(), o


def _host_table(table, shape, dtype, name):
    if torch.is_tensor(table):
        if table.is_cuda:
            raise ValueError('%s is a host table: reading it from the device would synchronise' % name)
        table = table.numpy()
    a = np.ascontiguousarray(np.asarray(table, dtype=dtype))
    if a.shape != shape:
        raise ValueError('%s must have shape %s, got %s' % (name, shape, a.shape))
    return a


def render_voxels(labels, origin, voxel_size, cameras, image_size, palette, shade=None, background=BACKGROUND,
                  want=('rgb',)):
    """Ray-cast the label volume for K cameras in one launch.

    labels uint8 [H, W, D] (CUDA); origin (x, y, z) metres of the grid's lowest corner; cameras: Camera(s) or rows
    [K, 16] (``Camera.row``); image_size (height, width), which the Camera objects are re-made at; palette RGBA [256, 4]
    (host); shade 6 floats in [0, 1] per face code (default ``SHADE``); background RGB.
    ``want`` picks the outputs: 'rgb' uint8 [K, h, w, 3], 'voxel' int32 [K, h, w] hit voxel index (h * W + w) * D + d or
    -1, 'face' int8 [K, h, w] face code or -1, 'dist' fp32 [K, h, w] hit depth or +inf.  Returns a dict of device
    tensors; nothing is read back to the host."""
    lib = _lib.load()
    labels, o = _grid(labels, origin)
    dev = labels.device
    h, w = int(image_size[0]), int(image_size[1])
    if isinstance(cameras, Camera):
        cameras = [cameras]
    if isinstance(cameras, (list, tuple)) and cameras and isinstance(cameras[0], Camera):
        cameras = [c.resized((h, w)) for c in cameras]
    cams = camera_rows(cameras, dev)
    K = cams.shape[0]
    pal = _host_table(palette, (256, 4), np.uint8, 'palette')
    sh = _host_table(SHADE if shade is None else shade, (6,), np.float32, 'shade')
    bg = _host_table(background, (3,), np.uint8, 'background')
    bad = set(want) - {'rgb', 'voxel', 'face', 'dist'}
    if bad or not want:
        raise ValueError('want must name some of rgb, voxel, face, dist; got %r' % (want,))
    out = {}
    if 'rgb' in want:
        out['rgb'] = torch.empty(K, h, w, 3, dtype=torch.uint8, device=dev)
    if 'voxel' in want:
        out['voxel'] = torch.empty(K, h, w, dtype=torch.int32, device=dev)
    if 'face' in want:
        out['face'] = torch.empty(K, h, w, dtype=torch.int8, device=dev)
    if 'dist' in want:
        out['dist'] = torch.empty(K, h, w, dtype=torch.float32, device=dev)
    H, W, D = labels.shape
    _lib.check(lib.so_voxel_render(_p(labels), H, W, D, o, float(voxel_size), _p(cams), K, h, w,
                                   pal.ctypes.data_as(C.c_void_p), sh.ctypes.data_as(C.c_void_p), bg.ctypes.data_as(C.c_void_p),
                                   _p(out.get('rgb')), _p(out.get('voxel')), _p(out.get('face')), _p(out.get('dist')),
                                   _stream()), 'so_voxel_render')
    return out


def drawn_table(palette=None):
    """uint8 [256]: 1 where the palette's alpha is non-zero (None: vis_3d.py's 0 < label < 100)."""
    if palette is None:
        return _drawn_labels().astype(np.uint8)
    return (_host_table(palette, (256, 4), np.uint8, 'palette')[:, 3] != 0).astype(np.uint8)


def voxel_mesh(labels, origin, voxel_size, palette=None):
    """The drawn voxels' exposed faces (the 6-neighbour is not drawn or lies outside the grid) as a mesh: each face 4
    vertices and 2 triangles, counter-clockwise seen from outside, in ascending voxel index then face code.  -> {'vertices'
    fp32 [4F, 3] metres, 'faces' int32 [2F, 3], 'normals' fp32 [4F, 3] outward unit, 'sem' uint8 [4F] the voxel's label};
    ``mesh.write_ply(path, m, colormap=palette)`` writes it.  Drawn: the palette's alpha, or 0 < label < 100 without
    one.  One synchronising read (the face count)."""
    lib = _lib.load()
    labels, o = _grid(labels, origin)
    dev = labels.device
    H, W, D = labels.shape
    drawn = drawn_table(palette)
    counts = torch.empty(H * W * D, dtype=torch.int32, device=dev)
    _lib.check(lib.so_voxel_faces_count(_p(labels), H, W, D, drawn.ctypes.data_as(C.c_void_p), _p(counts), _stream()),
               'so_voxel_faces_count')
    scans = torch.cumsum(counts, 0, dtype=torch.int32)
    n = int(scans[-1].item())                                                # the one host read
    if 4 * n >= 2 ** 31:
        raise _lib.SelfOccLibraryError('voxel_mesh: %d faces: vertex ids need more than int32' % n)
    m = dict(vertices=torch.empty(4 * n, 3, device=dev), faces=torch.empty(2 * n, 3, dtype=torch.int32, device=dev),
             normals=torch.empty(4 * n, 3, device=dev), sem=torch.empty(4 * n, dtype=torch.uint8, device=dev))
    if n:
        _lib.check(lib.so_voxel_faces_emit(_p(labels), H, W, D, o, float(voxel_size), drawn.ctypes.data_as(C.c_void_p),
                                           _p(scans), n, _p(m['vertices']), _p(m['faces']), _p(m['normals']), _p(m['sem']),
                                           _stream()), 'so_voxel_faces_emit')
    return m


# ---------------------------------------------------------------------------------------------------------------------
# files


def write_png(path, rgb):
    """Write an RGB image uint8 [h, w, 3] (array or tensor) as an 8-bit PNG with zlib and struct only."""
    if torch.is_tensor(rgb):
        rgb = rgb.detach().cpu().numpy()
    a = np.ascontiguousarray(rgb, dtype=np.uint8)
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError('write_png wants [h, w, 3], got %s' % (a.shape,))
    h, w, _ = a.shape
    raw = np.concatenate([np.zeros((h, 1), np.uint8), a.reshape(h, 3 * w)], 1).tobytes()   # filter type 0 per row

    def chunk(tag, data):
        return struct.pack('>I', len(data)) + tag + data + struct.pack('>I', zlib.crc32(tag + data) & 0xffffffff)

    with open(path, 'wb') as f:
        f.write(b'\x89PNG\r\n\x1a\n')
        f.write(chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 2, 0, 0, 0)))
        f.write(chunk(b'IDAT', zlib.compress(raw, 6)))
        f.write(chunk(b'IEND', b''))
