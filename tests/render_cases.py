"""Meshes, cameras and poses for the mesh-rendering tests (tests/test_render_cpu.py, tests/test_gpu_render.py) and
benchmarks/render.py.  Lengths are in millimetres, as in LINEMOD."""
import numpy as np

K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]], np.float32)


def icosphere(subdiv, radius=1.0):
    """A closed icosphere: 20 * 4^subdiv faces, outward winding, shared vertices."""
    p = (1 + 5 ** 0.5) / 2
    v = [(-1, p, 0), (1, p, 0), (-1, -p, 0), (1, -p, 0), (0, -1, p), (0, 1, p), (0, -1, -p), (0, 1, -p),
         (p, 0, -1), (p, 0, 1), (-p, 0, -1), (-p, 0, 1)]
    verts = [np.array(x, np.float64) / np.linalg.norm(x) for x in v]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2),
             (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11),
             (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    for _ in range(subdiv):
        cache = {}

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = verts[a] + verts[b]
                verts.append(m / np.linalg.norm(m))
                cache[key] = len(verts) - 1
            return cache[key]

        nxt = []
        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nxt += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nxt
    return (np.array(verts) * radius).astype(np.float32), np.array(faces, np.int32)


def cube(half=1.0):
    v = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32) * half
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                  [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    return v, f


def soup(n, rng, spread=60.0, size=25.0):
    """n random triangles around the origin, heavily overlapping."""
    c = rng.normal(0, spread, (n, 1, 3))
    v = (c + rng.normal(0, size, (n, 3, 3))).reshape(-1, 3).astype(np.float32)
    return v, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def poses(b, rng, depth=(600.0, 900.0), shift=40.0):
    """b random rotations in front of the camera: float32 [b,3,4]."""
    P = np.zeros((b, 3, 4), np.float32)
    for i in range(b):
        P[i, :, :3] = rotation(rng)
        P[i, :, 3] = (rng.normal(0, shift), rng.normal(0, shift), rng.uniform(*depth))
    return P


def camera_for(h, w, f=None):
    """A pinhole camera centred on an h x w image."""
    f = f if f is not None else 1.2 * max(h, w)
    return np.array([[f, 0, w / 2.0], [0, f, h / 2.0], [0, 0, 1]], np.float32)
