"""The Adam step on the H100 (DESIGN.md §19): pvnet_adam_step against oracle/adam_oracle.py bit for bit, against
torch.optim.Adam on CUDA, and pvnet_b200.optim.Adam inside real Resnet18_8s.forward_train steps: checkpoint swaps with
torch's Adam, a parameter without a gradient, launch count, no synchronisation, deterministic mode, streams."""
import copy

import numpy as np
import pytest
import torch

from oracle import adam_oracle as ao
from pvnet_b200 import _native, optim
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
HYPER = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)


def _native_step(tensors, step, dev=DEV, **kw):
    h = {**HYPER, **kw}
    optim._adam_step(torch.device(dev), tensors, h["lr"], h["betas"][0], h["betas"][1], h["eps"], h["weight_decay"],
                     step)


def _same_bits(t, want):
    """Equal as fp32 values, zeros by sign, NaN where the oracle has NaN (payloads are not compared)."""
    got = t.detach().cpu().numpy().reshape(-1)
    want = np.asarray(want, F32).reshape(-1)
    nan = np.isnan(want)
    return (np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan], want[~nan])
            and np.array_equal(np.signbit(got[~nan]), np.signbit(want[~nan])))


def _random_state(shapes, seed, dev=DEV):
    g = torch.Generator(device=dev).manual_seed(seed)
    ps = [torch.randn(s, device=dev, generator=g) for s in shapes]
    ms = [torch.randn(s, device=dev, generator=g) * 0.1 for s in shapes]
    vs = [torch.rand(s, device=dev, generator=g) * 0.01 for s in shapes]
    return g, ps, ms, vs


def _run_against_oracle(shapes, steps=5, first_step=1, seed=0, **kw):
    g, ps, ms, vs = _random_state(shapes, seed)
    want = [(p.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()) for p, m, v in zip(ps, ms, vs)]
    h = {**HYPER, **kw}
    for step in range(first_step, first_step + steps):
        gs = [torch.randn(s, device=DEV, generator=g) for s in shapes]
        _native_step(list(zip(ps, gs, ms, vs)), step, **kw)
        want = [ao.adam_step(P, gr.cpu().numpy(), M, V, step=step, **h) for (P, M, V), gr in zip(want, gs)]
        for i, ((P, M, V), p, m, v) in enumerate(zip(want, ps, ms, vs)):
            assert _same_bits(p, P) and _same_bits(m, M) and _same_bits(v, V), (step, i, shapes[i])


# ------------------------------------------------------------------ the kernel against the oracle

@pytest.mark.parametrize("numel", [1, 3, 20, 64, 4097, 2359296])
def test_kernel_equals_oracle(numel):
    _run_against_oracle([(numel,)], seed=numel)


@pytest.mark.parametrize("kw", [dict(weight_decay=1e-4), dict(betas=(0.3, 0.99)), dict(lr=0.0), dict(betas=(0.0, 0.0)),
                                dict(lr=3e-2, eps=1e-3, weight_decay=0.5)])
def test_kernel_equals_oracle_for_other_hyper_parameters(kw):
    """weight decay (the extra FMA), a lerp weight of 0.7 (ATen's other lerp form), and the corners of the ranges."""
    _run_against_oracle([(4097,), (64, 3, 7, 7)], first_step=7, **kw)


def _resnet_shapes():
    return [tuple(p.shape) for p in Resnet18_8s(ver_dim=18, seg_dim=2).parameters()]


def test_resnet18_8s_table_equals_oracle_in_one_launch():
    shapes = _resnet_shapes()
    assert len(shapes) == 77 and sum(int(np.prod(s)) for s in shapes) > 12_000_000
    _native.launch_count_reset()
    _run_against_oracle(shapes, steps=2, weight_decay=1e-4)
    assert _native.launch_count() == 2                    # one launch per step


def test_table_longer_than_one_launch():
    """The chunk boundary: tables of chunk, chunk + 1 and 2 * chunk + 3 non-empty tensors with empty entries in
    between take 1, 2 and 3 launches, and every tensor on either side of a boundary is stepped exactly once."""
    chunk = _native.lib().pvnet_adam_chunk_tensors()
    for n, launches in ((chunk, 1), (chunk + 1, 2), (2 * chunk + 3, 3)):
        shapes = [((i * 37) % 2500 + 1,) for i in range(n)]
        g, ps, ms, vs = _random_state(shapes, n)
        gs = [torch.randn(s, device=DEV, generator=g) for s in shapes]
        want = [ao.adam_step(p.cpu().numpy(), gr.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), step=2, **HYPER)
                for p, gr, m, v in zip(ps, gs, ms, vs)]
        table = []
        empty = torch.empty(0, device=DEV)
        for i, t in enumerate(zip(ps, gs, ms, vs)):
            if i % 50 == 0:
                table.append((empty, empty, empty, empty))
            table.append(t)
        _native.launch_count_reset()
        _native_step(table, 2)
        assert _native.launch_count() == launches
        for i, ((P, M, V), p, m, v) in enumerate(zip(want, ps, ms, vs)):
            assert _same_bits(p, P) and _same_bits(m, M) and _same_bits(v, V), (n, i)
    _native.launch_count_reset()
    _native_step([], 1)
    assert _native.launch_count() == 0


@pytest.mark.parametrize("numel", [5, 2048, 2049, 10001])
def test_unaligned_slice_gives_the_aligned_bits(numel):
    """Tensors that start 4 bytes into a 16-byte-aligned buffer take the scalar path; each of the four pointers in
    turn, and all of them."""
    g = torch.Generator(device=DEV).manual_seed(numel)
    base = [torch.randn(numel + 1, device=DEV, generator=g) for _ in range(4)]
    base[3] = base[3].abs() * 0.01
    ref = [t[1:].clone() for t in base]
    assert all(t.data_ptr() % 16 == 0 for t in ref)
    _native_step([(ref[0], ref[1], ref[2], ref[3])], 3, weight_decay=1e-4)
    P, M, V = ao.adam_step(*(t[1:].cpu().numpy() for t in base), step=3, **{**HYPER, "weight_decay": 1e-4})
    assert _same_bits(ref[0], P) and _same_bits(ref[2], M) and _same_bits(ref[3], V)
    for off in ([0], [1], [2], [3], [0, 1, 2, 3]):
        ts = []
        for i, t in enumerate(base):
            if i in off:
                ts.append(t.clone()[1:])
                assert ts[-1].data_ptr() % 16 == 4
            else:
                ts.append(t[1:].clone())
        _native_step([tuple(ts)], 3, weight_decay=1e-4)
        assert torch.equal(ts[0], ref[0]) and torch.equal(ts[2], ref[2]) and torch.equal(ts[3], ref[3]), off
        assert torch.equal(ts[1], base[1][1:])            # the gradient is only read


def test_special_values_propagate_as_the_oracle_says():
    inf, nan, sub = np.inf, np.nan, 1e-42
    cols = [  # p, g, m, v
        (1.0, 0.0, 0.0, 0.0), (1.0, -0.0, 0.0, 0.0), (-0.0, -0.0, -0.0, 0.0), (0.0, 0.0, 0.0, 0.0),
        (1.0, 1e-30, 0.0, sub), (1.0, -1e-30, 1e-35, sub), (1.0, 3e-21, 0.0, 0.0), (1.0, 0.0, 1e-3, sub),
        (1.0, 1e30, 0.0, 0.0), (1.0, -1e30, 0.0, 1e20), (1.0, inf, 0.0, 0.0), (1.0, -inf, 0.5, 0.1),
        (1.0, nan, 0.0, 0.0), (nan, 1.0, 0.0, 0.0), (1.0, 1.0, inf, 1.0), (1.0, 1.0, 1.0, inf), (3e38, -1.0, -1e30, 1e-30),
    ]
    for kw in (dict(), dict(weight_decay=0.1), dict(betas=(0.3, 0.99))):
        arr = np.array(cols, F32).T.copy()
        p, g, m, v = (torch.from_numpy(a.copy()).to(DEV) for a in arr)
        for step in (1, 2):
            _native_step([(p, g, m, v)], step, **kw)
            P, M, V = ao.adam_step(arr[0], arr[1], arr[2], arr[3], step=step, **{**HYPER, **kw})
            assert _same_bits(p, P) and _same_bits(m, M) and _same_bits(v, V), (kw, step)
            arr = np.stack([P, arr[1], M, V])
        assert np.isnan(P[10]) and np.isnan(P[12]) and np.isnan(P[13]) and np.isfinite(P[:8]).all()


# ------------------------------------------------------------------ against torch.optim.Adam on CUDA

SHAPES = [(64, 3, 7, 7), (64,), (4097,), (512, 512, 3, 3), (3,), (20, 32, 1, 1)]


def _params(seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, device=DEV, generator=g)) for s in SHAPES]


def _assert_same_optimizer_state(ps, opt, qs, ref, what=""):
    for i, (p, q) in enumerate(zip(ps, qs)):
        assert torch.equal(p, q), (what, "param", i)
        s, t = opt.state[p], ref.state[q]
        assert s.keys() == t.keys() == {"step", "exp_avg", "exp_avg_sq"}
        assert torch.equal(s["exp_avg"], t["exp_avg"]), (what, "exp_avg", i)
        assert torch.equal(s["exp_avg_sq"], t["exp_avg_sq"]), (what, "exp_avg_sq", i)
        assert s["step"].dtype == t["step"].dtype and s["step"].device == t["step"].device
        assert float(s["step"]) == float(t["step"]), (what, "step", i)


def _ten_steps(kw, check, **torch_kw):
    ps, qs = _params(), _params()
    opt, ref = optim.Adam(ps, lr=1e-3, **kw), torch.optim.Adam(qs, lr=1e-3, **torch_kw, **kw)
    g = torch.Generator(device=DEV).manual_seed(1)
    for step in range(1, 11):
        if step == 6:
            nu.set_learning_rate(opt, 2.5e-4)
            nu.set_learning_rate(ref, 2.5e-4)
        for p, q in zip(ps, qs):
            p.grad = torch.randn(p.shape, device=DEV, generator=g)
            q.grad = p.grad.clone()
        opt.step()
        ref.step()
        check(ps, opt, qs, ref, step)


KWS = [dict(), dict(weight_decay=1e-4), dict(betas=(0.3, 0.99), eps=1e-6)]


@pytest.mark.parametrize("kw", KWS)
def test_equals_torch_cuda_single_tensor_adam(kw):
    """Ten steps on the same inputs, the learning rate changed after the fifth: torch.equal in parameters and state
    with torch.optim.Adam(foreach=False), the sequence the kernel states."""
    _ten_steps(kw, _assert_same_optimizer_state, foreach=False)


@pytest.mark.parametrize("kw", KWS)
def test_close_to_torch_default_foreach_adam(kw):
    """torch's default on CUDA (foreach=True) is NOT bit-equal to its own foreach=False, and so not to the native
    step: it divides sqrt(v) by bias_correction2_sqrt where the single-tensor form multiplies by the reciprocal, which
    moves the denominator by an ulp.  The moments do not see the denominator and stay equal unless weight decay feeds
    the parameter back into the gradient (then: step + 1 ulps); the parameter is held to the accumulated rounding of
    its updates (each at most a few lr: 4 ulps of 10 lr plus one ulp of p per step).  Observed: at most 2.4e-7."""
    def check(ps, opt, qs, ref, step):
        for i, (p, q) in enumerate(zip(ps, qs)):
            for key in ("exp_avg", "exp_avg_sq"):
                s, t = opt.state[p][key], ref.state[q][key]
                if kw.get("weight_decay"):
                    s, t = s.cpu().numpy(), t.cpu().numpy()
                    assert np.all(np.abs(s - t) <= (step + 1) * np.spacing(np.abs(s))), (step, i, key)
                else:
                    assert torch.equal(s, t), (step, i, key)
            a, b = p.detach().cpu().numpy(), q.detach().cpu().numpy()
            assert np.all(np.abs(a - b) <= step * (np.spacing(np.abs(a)) + 4 * 2.0 ** -24 * 10 * 1e-3)), (step, i)
    _ten_steps(kw, check, foreach=True)


# ------------------------------------------------------------------ real training steps

def _batch(b=2, H=128, W=160, seed=0):
    rng = np.random.default_rng(seed)
    x = torch.randn(b, 3, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    mask = torch.from_numpy((rng.random((b, H, W)) < 0.3).astype(np.int64)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [W, H], (b, 9, 2)), np.ones((b, 9, 1))], 2)).to(DEV)
    return x, mask, hc


def _train_step(net, opt, batch):
    x, mask, hc = batch
    seg, ver = net.forward_train(x)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
    opt.zero_grad(set_to_none=True)
    (ls.mean() + lv.mean()).backward()
    opt.step()


def _twins():
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    return net, copy.deepcopy(net)


def _assert_same_training_state(net, opt, twin, ref, what=""):
    _assert_same_optimizer_state(list(net.parameters()), opt, list(twin.parameters()), ref, what)
    for (k, a), (_, b) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(a, b), (what, k)


def test_training_steps_equal_torch_adam_and_swap_through_state_dict(tmp_path):
    net, twin = _twins()
    opt, ref = optim.Adam(net.parameters(), lr=1e-3), torch.optim.Adam(twin.parameters(), lr=1e-3, foreach=False)
    for step in range(3):
        batch = _batch(seed=step)
        _train_step(net, opt, batch)
        _train_step(twin, ref, batch)
        _assert_same_training_state(net, opt, twin, ref, step)
    # swap mid-run through save_model / load_model: each network continues with the other optimizer
    nu.save_model(net, opt, 0, str(tmp_path / "native"))
    nu.save_model(twin, ref, 0, str(tmp_path / "torch"))
    opt2, ref2 = torch.optim.Adam(net.parameters(), lr=7.0, foreach=False), optim.Adam(twin.parameters(), lr=7.0)
    assert nu.load_model(net, opt2, str(tmp_path / "native")) == 1
    assert nu.load_model(twin, ref2, str(tmp_path / "torch")) == 1
    assert opt2.param_groups[0]["lr"] == ref2.param_groups[0]["lr"] == 1e-3
    opt2.param_groups[0]["foreach"] = False              # the native checkpoint carries no torch-only option
    batch = _batch(seed=3)
    _train_step(net, opt2, batch)
    _train_step(twin, ref2, batch)
    _assert_same_training_state(net, opt2, twin, ref2, "after the swap")
    assert float(opt2.state[net.convraw[3].bias]["step"]) == 4.0
    assert ref2.state[twin.convraw[3].bias]["step"].device.type == "cpu"


def test_parameter_without_gradient_is_left_alone():
    net, twin = _twins()
    opt, ref = optim.Adam(net.parameters(), lr=1e-3), torch.optim.Adam(twin.parameters(), lr=1e-3, foreach=False)
    _train_step(net, opt, _batch(seed=0))
    _train_step(twin, ref, _batch(seed=0))
    frozen = net.convraw[3].bias
    before = [frozen.detach().clone()] + [opt.state[frozen][k].clone() for k in ("exp_avg", "exp_avg_sq", "step")]
    for n, o in ((net, opt), (twin, ref)):
        n.convraw[3].bias.requires_grad_(False)
        _train_step(n, o, _batch(seed=1))
        n.convraw[3].bias.requires_grad_(True)
    assert frozen.grad is None
    after = [frozen.detach()] + [opt.state[frozen][k] for k in ("exp_avg", "exp_avg_sq", "step")]
    assert all(torch.equal(a, b) for a, b in zip(before, after)) and float(opt.state[frozen]["step"]) == 1.0
    assert float(opt.state[net.convraw[3].weight]["step"]) == 2.0
    _assert_same_training_state(net, opt, twin, ref, "frozen step")
    # the next step has two step values in one group: two calls, still torch's result
    _native.launch_count_reset()
    _train_step(net, opt, _batch(seed=2))
    _train_step(twin, ref, _batch(seed=2))
    _assert_same_training_state(net, opt, twin, ref, "mixed step values")
    assert float(opt.state[frozen]["step"]) == 2.0 and float(opt.state[net.convraw[3].weight]["step"]) == 3.0


def test_one_launch_no_synchronisation_and_deterministic():
    net, twin = _twins()
    opt, opt_twin = optim.Adam(net.parameters(), lr=1e-3), optim.Adam(twin.parameters(), lr=1e-3)
    batch = _batch(seed=5)
    _train_step(net, opt, batch)                          # creates the state
    _train_step(twin, opt_twin, batch)
    x, mask, hc = batch
    seg, ver = net.forward_train(x)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
    opt.zero_grad(set_to_none=True)
    (ls.mean() + lv.mean()).backward()
    torch.cuda.synchronize()
    n_params = sum(p.grad is not None for p in net.parameters())
    chunk = _native.lib().pvnet_adam_chunk_tensors()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    _native.launch_count_reset()
    try:
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert n_params == 77 and _native.launch_count() == -(-n_params // chunk) == 1
    # catch the twin up, then two seeded runs in deterministic mode give identical weights and state
    _train_step(twin, opt_twin, batch)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for seed in (6, 7):
            _train_step(net, opt, _batch(seed=seed))
            _train_step(twin, opt_twin, _batch(seed=seed))
    finally:
        torch.use_deterministic_algorithms(prev)
    _assert_same_training_state(net, opt, twin, opt_twin, "deterministic mode")


def test_step_on_a_side_stream_and_second_device():
    devs = [DEV] + (["cuda:1"] if torch.cuda.device_count() > 1 else [])
    for dev in devs:
        g = torch.Generator(device=dev).manual_seed(3)
        ps = [torch.nn.Parameter(torch.randn(s, device=dev, generator=g)) for s in SHAPES]
        qs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
        opt, ref = optim.Adam(ps, weight_decay=1e-4), torch.optim.Adam(qs, weight_decay=1e-4, foreach=False)
        side = torch.cuda.Stream(device=dev)
        for step in range(3):
            for p, q in zip(ps, qs):
                p.grad = torch.randn(p.shape, device=dev, generator=g)
                q.grad = p.grad.clone()
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):                 # the current device stays cuda:0 for dev = cuda:1's first step
                opt.step()
            torch.cuda.current_stream(dev).wait_stream(side)
            ref.step()
            _assert_same_optimizer_state(ps, opt, qs, ref, (dev, step))
    if len(devs) == 1:
        pytest.skip("one device: the second-device case did not run (the side-stream case passed)")
