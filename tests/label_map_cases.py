"""Cases for the label-map tests (tests/test_label_map_cpu.py, tests/test_gpu_label_map.py), the golden generator
tests/golden/make_golden_label_map.py and benchmarks/label_map.py.

* `golden_depth_maps(case)`: seeded stand-ins for what `OpenGLRenderer.render(class, pose, 'linemod')` returns to
  `get_mask_of_all_objects` (float32 [480,640] depth in metres, 0 where the object is not drawn), with overlaps,
  exact ties, values at and above the initial depth of 10, and missing poses.
* `scene(b, rng)`: nine overlapping icospheres at LINEMOD-like poses, in millimetres.
* `FakeOcclusionDB`: the parts of the reference's `OcclusionLineModDB` that `get_mask_of_all_objects` touches, over
  in-memory models and poses, with `OpenGLRenderer.render`'s depth path on the `lib.utils.opengl_render_backend`
  drop-in; `reference_loop` is that method's compositing, restated."""
import numpy as np

from tests import render_cases as rc

# OcclusionLineModDB.class_type_to_number (lib/utils/data_utils.py:685-695), in its order
OCCLUSION_CLASSES = (("ape", "001"), ("can", "004"), ("cat", "005"), ("driller", "006"), ("duck", "007"),
                     ("eggbox", "008"), ("glue", "009"), ("holepuncher", "010"), ("benchvise", "011"))
H, W = 480, 640
GOLDEN_CASES = 8
TIE_DEPTHS = np.float32([0.6, 0.75, 0.9, 1.0])


def golden_depth_maps(case):
    """-> [(class, depth f32 [480,640] or None for a missing pose)] in class order."""
    rng = np.random.default_rng(1000 + case)
    out = []
    r, c = np.mgrid[0:H, 0:W]
    for k, (name, _) in enumerate(OCCLUSION_CLASSES):
        if rng.random() < 0.2:
            out.append((name, None))
            continue
        d = np.zeros((H, W), np.float32)
        for _ in range(int(rng.integers(1, 4))):
            cy, cx = rng.uniform(100, 380), rng.uniform(120, 520)
            ry, rx = rng.uniform(20, 120), rng.uniform(20, 160)
            inside = ((r - cy) / ry) ** 2 + ((c - cx) / rx) ** 2 <= 1
            kind = rng.integers(0, 5)
            if kind == 0:                                   # one of a few values: exact ties between objects
                z = np.full((H, W), TIE_DEPTHS[rng.integers(0, len(TIE_DEPTHS))], np.float32)
            elif kind == 1:                                 # at or beyond the map's initial depth
                z = np.full((H, W), np.float32([10.0, 12.5])[rng.integers(0, 2)], np.float32)
            elif kind == 2:                                 # one ulp either side of a tie value
                base = TIE_DEPTHS[rng.integers(0, len(TIE_DEPTHS))]
                z = np.full((H, W), np.nextafter(base, np.float32(2 * (rng.random() < 0.5) - 1) * np.inf), np.float32)
            else:                                           # a plane: depth varies across the region
                z = (rng.uniform(0.4, 1.4) + rng.normal(0, 1e-3) * (c - cx) + rng.normal(0, 1e-3) * (r - cy))
                z = np.maximum(z, 0.05).astype(np.float32)
            d[inside] = z[inside]
        out.append((name, d))
    return out


def scene(b, rng, subdiv=5, per_image_k=True, absent=0.15):
    """Nine overlapping icospheres (20 * 4^subdiv faces each) at LINEMOD-like poses: meshes [(v, f)] * 9 in mm, labels,
    poses f32 [b,9,3,4] (t in mm), K [b,3,3] or [3,3], present u8 [b,9]."""
    meshes = [rc.icosphere(subdiv, r) for r in np.linspace(45.0, 95.0, 9)]
    labels = [int(n) for _, n in OCCLUSION_CLASSES]
    P = np.zeros((b, 9, 3, 4), np.float32)
    for i in range(b):
        centre = np.array([rng.normal(0, 60), rng.normal(0, 40), rng.uniform(650, 950)])
        for m in range(9):
            P[i, m, :, :3] = rc.rotation(rng)
            P[i, m, :, 3] = centre + np.array([rng.normal(0, 60), rng.normal(0, 50), rng.normal(0, 60)])
    if per_image_k:
        K = np.stack([rc.K_LINEMOD] * b).astype(np.float64)
        K[:, 0, 0] += rng.normal(0, 5, b)
        K[:, 1, 1] += rng.normal(0, 5, b)
        K[:, :2, 2] += rng.normal(0, 4, (b, 2))
        K = K.astype(np.float32)
    else:
        K = rc.K_LINEMOD
    present = (rng.random((b, 9)) >= absent).astype(np.uint8)
    return meshes, labels, P, K, present


class FakeRenderer:
    """`OpenGLRenderer`'s interface over in-memory models; `render` is its depth path (render_utils.py:510-524) on the
    `lib.utils.opengl_render_backend` drop-in."""
    intrinsic_matrix = {"linemod": rc.K_LINEMOD.astype(np.float64)}

    def __init__(self, models):
        self.models = models
        self.loads = 0

    def load_ply(self, class_type, color=None):
        self.loads += 1
        return self.models[class_type]

    def render(self, class_type, pose, camera_type=None, intrinsic_matrix=None, render_type="depth", color=None):
        from lib.utils.opengl_render_backend import render
        assert render_type == "depth"
        model = self.load_ply(class_type)
        K = self.intrinsic_matrix[camera_type] if camera_type is not None else intrinsic_matrix
        R, t = pose[:, :3], pose[:, 3:] * 1000.
        return render(model, im_size=[640, 480], K=K, R=R, t=t, clip_near=10, clip_far=10000, mode="depth") / 1000.


class FakeOcclusionDB:
    """What get_mask_of_all_objects reads of an OcclusionLineModDB: poses[(class, index)] holds [3,4] arrays (metres;
    a missing key reads as the empty array of a missing pose file)."""
    class_type_to_number = dict(OCCLUSION_CLASSES)

    def __init__(self, models, poses):
        self.class_type = None
        self.opengl_renderer = FakeRenderer(models)
        self.poses = poses

    def read_blender_pose(self, index):
        return self.poses.get((self.class_type, index), np.array([]))


def fake_db(indices, rng, subdiv=3):
    """Nine icosphere models (mm, colours in 0..255 as a PLY gives them) and their poses at `indices`: float64
    poses, float32 for benchvise (read_benchvise_pose returns float32), and some missing."""
    models = {}
    for k, ((name, _), r) in enumerate(zip(OCCLUSION_CLASSES, np.linspace(45.0, 95.0, 9))):
        v, f = rc.icosphere(subdiv, r)
        models[name] = {"pts": v.astype(np.float64), "faces": f.astype(np.int64),
                        "colors": rng.uniform(0, 255, (len(v), 3))}
    poses = {}
    for index in indices:
        centre = np.array([rng.normal(0, 0.06), rng.normal(0, 0.04), rng.uniform(0.65, 0.95)])
        for name, _ in OCCLUSION_CLASSES:
            if rng.random() < 0.15:
                continue
            pose = np.concatenate([rc.rotation(rng), (centre + rng.normal(0, 0.05, 3))[:, None]], 1)
            poses[(name, index)] = pose.astype(np.float32) if name == "benchvise" else pose
    return FakeOcclusionDB(models, poses)


def reference_loop(db, index):
    """get_mask_of_all_objects' compositing: a map of zeros and a depth map of 10; object by object in
    class_type_to_number order, each pixel its render draws (depth != 0) nearer than the map takes its number."""
    mask_map = np.zeros((H, W), np.uint8)
    depth_map = 10 * np.ones((H, W), np.float32)
    for class_type in db.class_type_to_number.keys():
        db.class_type = class_type
        pose = db.read_blender_pose(index)
        if len(pose) == 0:
            continue
        depth = db.opengl_renderer.render(class_type, pose, camera_type="linemod")
        take = (depth != 0) & (depth < depth_map)
        mask_map[take] = int(db.class_type_to_number[class_type])
        depth_map[take] = depth[take]
    return mask_map
