"""CPU: the validation-loss oracle (oracle/loss_oracle.py) against hand-computed cases and against the reference's own
smooth_l1_loss / compute_precision_recall (tests/golden/ref_net_utils.npz, tests/golden/make_golden_net_utils.py);
the grad-mode torch expressions of pvnet_b200/net_utils.py against the same record; the `lib.utils.net_utils` shim's
import lines, signatures and host-side helpers; and the C ABI's argument checks."""
import ctypes
import inspect
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import loss_oracle as lo
from pvnet_b200 import _native
from pvnet_b200 import net_utils as nu
from tests.helpers import GOLDEN, same_as_stored
from tests.loss_cases import CASES, canon_nan, case_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_net_utils.npz")))


# ------------------------------------------------------------------------------------------------------ oracle
def test_oracle_smooth_l1_hand_computed():
    # sigma = 1: c1 = 1, c2 = 0.5, c3 = 0.5; |d| < 1 -> d^2/2, else |d| - 1/2
    pred = np.array([0.5, -2.0, 3.0, 0.0], np.float32).reshape(1, 4, 1, 1)
    tgt = np.array([0.0, 0.0, 1.0, 0.0], np.float32).reshape(1, 4, 1, 1)
    w = np.ones((1, 1, 1, 1), np.float32)
    el = lo.smooth_l1_elementwise(pred, tgt, w, 1.0).ravel()
    assert el.tolist() == [0.125, 1.5, 1.5, 0.0]
    # sigma = 2: c1 = 0.25, c2 = 2, c3 = 0.125; weight 0.5 halves the difference
    el2 = lo.smooth_l1_elementwise(pred, tgt, np.full((1, 1, 1, 1), 0.5, np.float32), 2.0).ravel()
    assert el2.tolist() == [2 * 0.25 ** 2, 1.0 - 0.125, 1.0 - 0.125, 0.0]
    norm = lo.smooth_l1_normalized(pred, tgt, w, 1.0)
    assert norm.dtype == np.float32 and norm[0] == np.float32(3.125) / (np.float32(4) + np.float32(1e-3))
    # an infinite difference gives inf * 0 = NaN in the quadratic branch, as torch
    inf = lo.smooth_l1_elementwise(np.full((1, 1, 1, 1), np.inf, np.float32), np.zeros((1, 1, 1, 1), np.float32),
                                   w, 1.0)
    assert np.isnan(inf).all()


def test_oracle_cross_entropy_hand_computed():
    seg = np.array([[[[0.0, 2.0, 1.0]], [[0.0, 0.0, 1.0]]]], np.float32)      # [1,2,1,3]
    mask = np.array([[[0, 1, -100]]])
    want = (np.log(2.0) + (np.log(1 + np.exp(2.0)) - 0.0) + 0.0) / 3
    assert np.isclose(lo.cross_entropy(seg, mask)[0], want, rtol=1e-7)
    assert np.isnan(lo.cross_entropy(seg, np.array([[[0, 2, 0]]]))[0])          # target 2 with C = 2
    assert np.isnan(lo.cross_entropy(seg, np.array([[[0, -1, 0]]]))[0])


def test_oracle_argmax_and_counts_hand_computed():
    nan = np.nan
    seg = np.array([[[[1, 2, nan, 5, nan]], [[1, 1, 0, nan, nan]], [[0, 2, 9, 5, 0]]]], np.float32)   # [1,3,1,5]
    assert lo.argmax(seg).ravel().tolist() == [0, 0, 0, 1, 0]     # ties -> first; NaN wins; first NaN
    mask = np.array([[[1, 0, 2, 1, 0]]])
    tp, fp, fn = lo.precision_recall_counts(seg, mask)
    assert (tp[0], fp[0], fn[0]) == (1, 0, 3)                      # p = [0,0,0,1,0], t = [1,0,2,1,0]
    p, r = lo.precision_recall(seg, mask)
    assert p[0] == 1 and r[0] == np.float32(2) / np.float32(5)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_reference_golden(name):
    g = _golden()
    seg, mask, pred, vertex, weights, sigma = case_inputs(name)
    assert same_as_stored(canon_nan(lo.smooth_l1_elementwise(pred, vertex, weights, sigma)), g[f"{name}/elem"])
    np.testing.assert_allclose(lo.smooth_l1_normalized(pred, vertex, weights, sigma), g[f"{name}/norm"], rtol=1e-6)
    p, r = lo.precision_recall(seg, mask)
    assert p.tobytes() == g[f"{name}/precision"].tobytes() and r.tobytes() == g[f"{name}/recall"].tobytes()


@pytest.mark.parametrize("name", list(CASES))
def test_torch_expressions_equal_reference_golden(name):
    """The grad-mode path (CPU tensors that require grad) against the reference's record and the oracle."""
    g = _golden()
    seg, mask, pred, vertex, weights, sigma = case_inputs(name)
    p = torch.from_numpy(pred).requires_grad_()
    el = nu.smooth_l1_loss(p, torch.from_numpy(vertex), torch.from_numpy(weights), sigma=sigma, normalize=False)
    assert same_as_stored(canon_nan(el), g[f"{name}/elem"])
    norm = nu.smooth_l1_loss(p, torch.from_numpy(vertex), torch.from_numpy(weights), sigma=sigma)
    np.testing.assert_allclose(norm.detach().numpy(), g[f"{name}/norm"], rtol=1e-6)
    s = torch.from_numpy(seg).requires_grad_()
    prec, rec = nu.compute_precision_recall(s, torch.from_numpy(mask))
    assert prec.numpy().tobytes() == g[f"{name}/precision"].tobytes()
    assert rec.numpy().tobytes() == g[f"{name}/recall"].tobytes()
    ce = nu._cross_entropy_torch(s, torch.from_numpy(mask)).detach().numpy()
    np.testing.assert_allclose(ce, lo.cross_entropy(seg, mask), rtol=1e-5)


def test_torch_cross_entropy_ignore_and_invalid():
    seg = torch.randn(2, 2, 4, 4, generator=torch.Generator().manual_seed(0)).requires_grad_()
    mask = torch.randint(0, 2, (2, 4, 4), generator=torch.Generator().manual_seed(1))
    mask[0, 0, :2] = -100
    mask[1, 2, 3] = 5
    got = nu._cross_entropy_torch(seg, mask).detach().numpy()
    want = lo.cross_entropy(seg.detach().numpy(), mask.numpy())
    assert np.isnan(got[1]) and np.isnan(want[1])
    np.testing.assert_allclose(got[0], want[0], rtol=1e-6)


def test_cpu_tensors_without_grad_raise():
    seg, mask, pred, vertex, weights, _ = (torch.from_numpy(a) if isinstance(a, np.ndarray) else a
                                           for a in case_inputs("k9_s1_binary"))
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.smooth_l1_loss(pred, vertex, weights)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.compute_precision_recall(seg, mask)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            nu.seg_vertex_losses(seg, pred.requires_grad_(), mask, vertex, weights)


def test_rejected_shapes_and_dtypes():
    pred = torch.zeros(2, 4, 5, 6)
    with pytest.raises(ValueError, match=r"\[b,1,h,w\]"):
        nu.smooth_l1_loss(pred, pred, torch.zeros(2, 4, 5, 6))
    with pytest.raises(ValueError, match=r"\[b,1,h,w\]"):
        nu.smooth_l1_loss(pred, pred, torch.zeros(1, 1, 5, 6))
    with pytest.raises(ValueError, match="float32"):
        nu.smooth_l1_loss(pred.double(), pred.double(), torch.zeros(2, 1, 5, 6, dtype=torch.float64))
    with pytest.raises(ValueError, match="float32"):
        nu.compute_precision_recall(torch.zeros(2, 2, 5, 6, dtype=torch.float16), torch.zeros(2, 5, 6, dtype=torch.long))
    with pytest.raises(ValueError, match="mask"):
        nu.compute_precision_recall(torch.zeros(2, 2, 5, 6), torch.zeros(2, 5, 6))


# ------------------------------------------------------------------------------------------------------- shim
def test_reference_import_lines_without_optional_packages():
    code = "\n".join([
        "import sys",
        "from lib.utils.net_utils import smooth_l1_loss, load_model, compute_precision_recall",      # tools/demo.py:6
        "from lib.utils.net_utils import AverageMeter, Recorder, smooth_l1_loss, load_model, save_model, "
        "adjust_learning_rate, compute_precision_recall, set_learning_rate",                        # train_linemod.py:19
        "print(sorted(m for m in ('tensorboardX', 'easydict', 'torchvision') if m in sys.modules))",
    ])
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "[]", out.stdout


def _signature(fn):
    parts = []
    for p in inspect.signature(fn).parameters.values():
        parts.append(p.name if p.default is inspect.Parameter.empty else f"{p.name}={p.default!r}")
    return ", ".join(parts)


def test_signatures_equal_reference():
    import lib.utils.net_utils as shim
    with open(os.path.join(GOLDEN, "ref_net_utils_signatures.json")) as f:
        expected = json.load(f)
    assert len(expected) == 14
    for name, want in expected.items():
        if "." in name:
            cls, meth = name.split(".")
            fn = getattr(getattr(shim, cls), meth)
        else:
            fn = getattr(shim, name)
        assert _signature(fn) == want, name


def test_average_meter():
    m = nu.AverageMeter()
    assert isinstance(m, dict) and (m.val, m.avg, m.sum, m.count) == (0, 0, 0, 0)
    m.update(2.0, n=3)
    m.update(4.0)
    assert m.val == 4.0 and m.sum == 10.0 and m.count == 4 and m.avg == 2.5 and m["avg"] == 2.5
    m.reset()
    assert m == {"val": 0, "avg": 0, "sum": 0, "count": 0}
    with pytest.raises(AttributeError):
        m.missing


def test_save_load_model_round_trip(tmp_path, capsys):
    net = torch.nn.Linear(3, 2)
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
    net(torch.ones(1, 3)).sum().backward()
    opt.step()
    d = str(tmp_path / "a" / "b")
    assert nu.load_model(net, opt, d) == 0                        # no directory
    nu.save_model(net, opt, 3, d)
    nu.save_model(net, opt, 12, d)
    assert sorted(os.listdir(d)) == ["12.pth", "3.pth"]
    net2 = torch.nn.Linear(3, 2)
    opt2 = torch.optim.SGD(net2.parameters(), lr=0.5, momentum=0.9)
    assert nu.load_model(net2, opt2, d) == 13                     # latest epoch + 1
    assert torch.equal(net2.weight, net.weight) and opt2.param_groups[0]["lr"] == 0.1
    assert nu.load_model(net2, opt2, d, epoch=3) == 4
    assert "epoch 3" in capsys.readouterr().out
    os.makedirs(tmp_path / "empty")
    assert nu.load_model(net2, opt2, str(tmp_path / "empty")) == 0


def test_learning_rate_helpers():
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.1)
    nu.adjust_learning_rate(opt, 0, 0.5, 2)                        # (0+1) % 2 != 0: unchanged
    assert opt.param_groups[0]["lr"] == 0.1
    nu.adjust_learning_rate(opt, 1, 0.5, 2)
    assert opt.param_groups[0]["lr"] == 0.05
    nu.adjust_learning_rate(opt, 3, 1e-6, 2, min_lr=1e-3)
    assert opt.param_groups[0]["lr"] == 1e-3
    nu.set_learning_rate(opt, 0.25)
    assert opt.param_groups[0]["lr"] == 0.25


def test_recorder_without_writer(tmp_path, capsys):
    dump = str(tmp_path / "log.txt")
    r = nu.Recorder(rec=False, dump_fn=dump)
    r.rec_loss(0.5, 7, name="val/loss")
    r.rec_loss_batch({"val/scalar/seg": 0.25, "val/scalar/ver": 1.0}, 3, 2, prefix="val")
    r.rec_segmentation(torch.zeros(1, 2, 4, 4), 2, 1, 0)              # no writer: nothing to log, nothing imported
    r.rec_vertex(torch.zeros(1, 2, 4, 4), torch.zeros(1, 1, 4, 4), 1, 0)
    lines = open(dump).read().splitlines()
    assert lines[0] == "val/loss 7 0.5"
    assert lines[1] == "val epoch 2 step 3 seg 0.25000000  ver 1.00000000 "
    assert capsys.readouterr().out.splitlines() == lines


def test_recorder_with_stub_tensorboardx(monkeypatch, tmp_path):
    calls = []

    class SummaryWriter:
        def __init__(self, log_dir=None):
            calls.append(("init", log_dir))

        def add_scalar(self, *a):
            calls.append(("scalar",) + a)

    stub = types.ModuleType("tensorboardX")
    stub.SummaryWriter = SummaryWriter
    monkeypatch.setitem(sys.modules, "tensorboardX", stub)
    r = nu.Recorder(True, str(tmp_path), None)
    r.rec_loss(1.5, 2)
    r.rec_loss_batch({"train/scalar/seg": 0.5}, 4, 1)
    assert calls == [("init", str(tmp_path)), ("scalar", "data/loss", 1.5, 2), ("scalar", "train/scalar/seg", 0.5, 4)]


def test_recorder_without_tensorboardx_raises_import_error(monkeypatch):
    monkeypatch.setitem(sys.modules, "tensorboardX", None)
    with pytest.raises(ImportError, match="tensorboardX"):
        nu.Recorder(rec=True)


# -------------------------------------------------------------------------------------------------------- ABI
def test_abi_argument_validation():
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_seg_vertex_losses_workspace_bytes(16, 480, 640, ctypes.byref(n)) == 0 and n.value > 0
    assert L.pvnet_seg_vertex_losses_workspace_bytes(0, 480, 640, ctypes.byref(n)) == -1
    assert b"dimension" in L.pvnet_last_error()
    s4 = (ctypes.c_int64 * 4)(20 * 64, 64, 8, 1)
    s3 = (ctypes.c_int64 * 3)(64, 8, 1)
    bad4 = (ctypes.c_int64 * 4)(20 * 64, 64, 8, 2)
    p = ctypes.c_void_p(256)                                       # never dereferenced: every call below is refused
    out = ctypes.c_void_p(512)

    def call(seg=p, segs=s4, mask=p, msz=8, masks=s3, pred=p, preds=s4, tgt=p, tgts=s4, wgt=p, wgts=s4, b=2, h=8,
             w=8, C=2, vd=18, sigma=1.0, ls=out, lv=out, pr=out, rc=out, ws=p, wsb=1 << 20):
        return L.pvnet_seg_vertex_losses(seg, segs, mask, msz, masks, pred, preds, tgt, tgts, wgt, wgts, b, h, w, C,
                                         vd, sigma, 1, ls, lv, pr, rc, ws, wsb, None)

    cases = [
        (dict(b=0), b"dimension"), (dict(h=-1), b"dimension"), (dict(C=0), b"dimension"), (dict(vd=0), b"dimension"),
        (dict(seg=None), b"null"), (dict(mask=None), b"null"), (dict(pred=None), b"null"), (dict(wgt=None), b"null"),
        (dict(ws=None), b"null"), (dict(masks=None), b"null"),
        (dict(segs=bad4), b"unit stride"), (dict(tgts=bad4), b"unit stride"), (dict(wgts=bad4), b"unit stride"),
        (dict(msz=2), b"mask_elem_size"), (dict(wsb=8), b"workspace"), (dict(sigma=0.0), b"sigma"),
        (dict(ls=None, lv=None, pr=None, rc=None), b"no output"),
    ]
    for kw, text in cases:
        assert call(**kw) == -1, kw
        assert text in L.pvnet_last_error(), (kw, L.pvnet_last_error())
