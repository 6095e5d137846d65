"""Regenerates tests/golden/ref_render.npz and tests/golden/ref_render_signature.json from the reference's
lib/utils/opengl_render_backend.py:

* the positional parameters of its `render` (names and default expressions), read with `ast`;
* for a few K, R, t, image sizes and clip planes, the matrices its own `render` builds -- the model-view, the
  projection (`_compute_calib_proj`) and their product -- with glumpy replaced in sys.modules by a stub that runs the
  draw callback once and records what `draw_depth` receives instead of drawing.

tests/test_render_cpu.py restates GL's clip -> NDC -> viewport -> row-flip chain on these matrices.
    PVNET_REFERENCE=<path> python tests/golden/make_golden_render.py
"""
import ast
import importlib.util
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SOURCE = "lib/utils/opengl_render_backend.py"


def signature(fn):
    args = fn.args.args
    defaults = [None] * (len(args) - len(fn.args.defaults)) + list(fn.args.defaults)
    return ", ".join(a.arg if d is None else f"{a.arg}={ast.unparse(d)}" for a, d in zip(args, defaults))


def stub_glumpy():
    """A glumpy with just what the module touches at import and in `render` outside the draw functions."""
    glumpy = types.ModuleType("glumpy")
    app, gloo, gl, log = (types.ModuleType("glumpy." + n) for n in ("app", "gloo", "gl", "log"))

    class Window:
        def __init__(self, **kw):
            self.handler = None

        def event(self, fn):
            self.handler = fn
            Window.last = self
            return fn

        def clear(self):
            pass

        def close(self):
            pass

    app.use = lambda name: None
    app.Window = Window
    app.run = lambda framecount=0: Window.last.handler(0.0)
    gloo.VertexBuffer = type("VertexBuffer", (np.ndarray,), {})
    gloo.IndexBuffer = type("IndexBuffer", (np.ndarray,), {})
    log.log = types.SimpleNamespace(setLevel=lambda level: None)
    glumpy.app, glumpy.gloo, glumpy.gl, glumpy.log = app, gloo, gl, log
    for name, mod in (("glumpy", glumpy), ("glumpy.app", app), ("glumpy.gloo", gloo), ("glumpy.gl", gl),
                      ("glumpy.log", log)):
        sys.modules[name] = mod


def rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


CASES = [
    # name, K, im_size [w, h], t shape, clip_near, clip_far
    ("linemod", [[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]], (640, 480), (3, 1), 100, 2000),
    ("skew_t3", [[600.0, 3.5, 310.0], [0, 590.0, 250.0], [0, 0, 1]], (640, 480), (3,), 50, 3000),
    ("odd_size", [[90.0, 0, 20.5], [0, 85.0, 15.25], [0, 0, 1]], (37, 29), (3, 1), 10, 500),
    ("tall", [[300.0, 0, 60.0], [0, 310.0, 160.0], [0, 0, 1]], (121, 333), (3,), 1, 100),
]


def main():
    sys.path.insert(0, ROOT)
    from tests.helpers import GOLDEN, reference_root
    path = os.path.join(reference_root(), SOURCE)
    tree = ast.parse(open(path).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "render")
    with open(os.path.join(GOLDEN, "ref_render_signature.json"), "w") as f:
        json.dump({"render": signature(fn)}, f, indent=1, sort_keys=True)
        f.write("\n")

    stub_glumpy()
    spec = importlib.util.spec_from_file_location("ref_opengl_render_backend", path)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    seen = {}

    def record(shape, vertex_buffer, index_buffer, mat_model, mat_view, mat_proj):
        seen.update(shape=shape, mv=ref._compute_model_view(mat_model, mat_view),
                    mvp=ref._compute_model_view_proj(mat_model, mat_view, mat_proj), proj=mat_proj)
        return np.zeros(shape, np.float32)

    ref.draw_depth = record
    rng = np.random.default_rng(7)
    model = {"pts": np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), "faces": np.array([[0, 1, 2]])}
    out = {}
    for name, K, im_size, tshape, near, far in CASES:
        R = rotation(rng)
        t = np.array([rng.normal(0, 40), rng.normal(0, 40), rng.uniform(2, 5) * near]).reshape(tshape)
        K = np.array(K)
        ref.render(model, im_size, K, R, t, clip_near=near, clip_far=far, mode="depth")
        assert seen["shape"] == (im_size[1], im_size[0])
        for k, v in (("K", K), ("R", R), ("t", t), ("im_size", np.array(im_size)), ("clip", np.array([near, far])),
                     ("mv", seen["mv"]), ("proj", seen["proj"]), ("mvp", seen["mvp"])):
            out[f"{name}/{k}"] = v
    np.savez(os.path.join(GOLDEN, "ref_render.npz"), **out)
    print("wrote", len(CASES), "cases")


if __name__ == "__main__":
    main()
