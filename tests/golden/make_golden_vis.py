"""Generate tests/golden/reference_golden_vis.npz from the reference's 3D visualisation (vis_3d.py, vis_pics.py).

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored arrays):
    python tests/golden/make_golden_vis.py <path to the SelfOcc checkout>
mayavi cannot be imported without a display, so nothing is imported: the scripts are parsed with ``ast``, and only two
self-contained functions (``get_grid_coords``, ``create_label_colormap``) are compiled from their parsed definitions and
run with numpy.  Stored:
* nuscenes_colors [16, 4]: the RGBA table ``draw`` assigns to the glyphs' lookup table for nuScenes;
* kitti_colors [19, 3]: ``create_label_colormap()``;
* sem_vmax_kitti / sem_vmax_nuscenes, sem_vmin: the scalar range of the semantic glyphs;
* drawn_lo / drawn_hi: the label window ``(label > lo) & (label < hi)`` of the drawn voxels;
* grid_coords [N, 3] and grid_dims / grid_res: ``get_grid_coords(dims, res)`` for a small square grid;
* cam_position / cam_focal_point / cam_view_up / cam_view_angle / cam_clip: the nuScenes camera set last in ``draw``,
  and cam_elevations: the Elevation angles applied after it, in order.
"""
import ast
import os
import sys
import numpy as np

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)
HERE = os.path.dirname(os.path.abspath(__file__))
GRID_DIMS = (5, 5, 3)
GRID_RES = (0.4, 0.4, 0.4)


def _parse(name):
    with open(os.path.join(REF, name)) as f:
        return ast.parse(f.read())


def _function(tree, name):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)


def _compile(fn):
    ns = {'np': np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), '<reference>', 'exec'), ns)
    return ns[fn.name]


def _attr_path(node):
    out = []
    while isinstance(node, ast.Attribute):
        out.append(node.attr)
        node = node.value
    if isinstance(node, ast.Name):
        out.append(node.id)
    return '.'.join(reversed(out))


def main():
    if REF is None:
        sys.exit(__doc__)
    vis = _parse('vis_3d.py')
    pics = _parse('vis_pics.py')
    draw = _function(vis, 'draw')

    # the nuScenes colour table: the np.array(...) literal of rows of 4 integers inside draw
    nusc = None
    for n in ast.walk(draw):
        if isinstance(n, ast.Call) and _attr_path(n.func) == 'np.array' and n.args and isinstance(n.args[0], ast.List):
            rows = ast.literal_eval(n.args[0])
            if rows and all(len(r) == 4 for r in rows):
                nusc = np.array(rows, dtype=np.uint8)
    assert nusc is not None and nusc.shape == (16, 4), nusc

    # the semantic glyphs' vmin / vmax and the drawn-label window
    vmin = vmax_k = vmax_n = None
    for n in ast.walk(draw):
        if isinstance(n, ast.keyword) and n.arg == 'vmin':
            vmin = ast.literal_eval(n.value)
        if isinstance(n, ast.keyword) and n.arg == 'vmax' and isinstance(n.value, ast.IfExp):
            vmax_k, vmax_n = ast.literal_eval(n.value.body), ast.literal_eval(n.value.orelse)
    lo = hi = None
    for n in ast.walk(draw):
        if isinstance(n, ast.Compare) and len(n.ops) == 1 and isinstance(n.comparators[0], ast.Constant):
            if isinstance(n.ops[0], ast.Gt) and n.comparators[0].value == 0 and lo is None:
                lo = 0
            if isinstance(n.ops[0], ast.Lt) and hi is None:
                hi = n.comparators[0].value
    assert None not in (vmin, vmax_k, vmax_n, lo, hi)

    kitti = _compile(_function(pics, 'create_label_colormap'))()
    coords = _compile(_function(vis, 'get_grid_coords'))(list(GRID_DIMS), list(GRID_RES))

    # the nuScenes camera: the statements after the last `scene.camera.position = ...` of the nuScenes branch
    branch = next(n for n in ast.walk(draw) if isinstance(n, ast.If) and isinstance(n.test, ast.Compare)
                  and isinstance(n.test.comparators[0], ast.Constant) and n.test.comparators[0].value == 'nuscenes')
    body = [s for s in branch.body]
    last = max(i for i, s in enumerate(body) if isinstance(s, ast.Assign)
               and _attr_path(s.targets[0]) == 'scene.camera.position')
    cam, elevations = {}, []
    for s in body[last:]:
        if isinstance(s, ast.Assign):
            cam[_attr_path(s.targets[0]).split('.')[-1]] = ast.literal_eval(s.value)
        elif isinstance(s, ast.Expr) and isinstance(s.value, ast.Call) and _attr_path(s.value.func) == 'scene.camera.elevation':
            elevations.append(ast.literal_eval(s.value.args[0]))

    out = os.path.join(HERE, 'reference_golden_vis.npz')
    np.savez_compressed(
        out, nuscenes_colors=nusc, kitti_colors=np.asarray(kitti, dtype=np.uint8), sem_vmin=np.int64(vmin),
        sem_vmax_kitti=np.int64(vmax_k), sem_vmax_nuscenes=np.int64(vmax_n), drawn_lo=np.int64(lo), drawn_hi=np.int64(hi),
        grid_coords=np.asarray(coords, dtype=np.float32), grid_dims=np.array(GRID_DIMS), grid_res=np.array(GRID_RES),
        cam_position=np.array(cam['position'], dtype=np.float64), cam_focal_point=np.array(cam['focal_point'], dtype=np.float64),
        cam_view_up=np.array(cam['view_up'], dtype=np.float64), cam_view_angle=np.float64(cam['view_angle']),
        cam_clip=np.array(cam['clipping_range'], dtype=np.float64), cam_elevations=np.array(elevations, dtype=np.float64))
    print('wrote', out, 'elevations', elevations)


if __name__ == '__main__':
    main()
