"""CPU: the Adam step's oracle, the drop-in optimizer's state and refusals, and pvnet_adam_step's argument checks
(DESIGN.md §19).  Nothing here launches a kernel; the binding comparisons (kernel against oracle bit for bit, kernel
against torch's CUDA Adam) are tests/test_gpu_adam.py."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import adam_oracle as ao
from pvnet_b200 import _native, net_utils, optim

F32 = np.float32


# ------------------------------------------------------------------ the oracle

def _round_f32(x: Fraction):
    """The fp32 nearest (ties to even) to the rational x, by exact arithmetic on the two neighbours."""
    lo = F32(float(x))                                    # within an ulp or so of x: a starting point
    while Fraction(float(lo)) > x:
        lo = np.nextafter(lo, F32(-np.inf))
    while Fraction(float(np.nextafter(lo, F32(np.inf)))) <= x:
        lo = np.nextafter(lo, F32(np.inf))
    hi = np.nextafter(lo, F32(np.inf))
    dl, dh = x - Fraction(float(lo)), Fraction(float(hi)) - x
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (lo.view(np.uint32) & 1) == 0 else hi


def test_oracle_fma_rounds_once():
    # the case a sum in fp64 rounded again to fp32 gets wrong: 1 + 2^-24 + 2^-60 lies above the tie
    a, b = F32(2.0 ** -12 + 2.0 ** -30), F32(2.0 ** -12 + 2.0 ** -31)
    exact = Fraction(float(a)) * Fraction(float(b)) + 1
    assert ao.fma(a, b, F32(1)) == _round_f32(exact)
    rng = np.random.default_rng(0)
    a = rng.standard_normal(400).astype(F32)
    b = rng.standard_normal(400).astype(F32)
    c = -(a * b) * F32(1 + 2.0 ** -20)                    # heavy cancellation: the low product bits decide
    c[::4] = rng.standard_normal(100).astype(F32) * F32(1e-30)
    a[1::4] *= F32(1e-25)                                 # subnormal results
    c[1::4] *= F32(1e-25)
    got = ao.fma(a, b, c)
    for x, y, z, r in zip(a, b, c, got):
        assert r == _round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
    assert np.isnan(ao.fma(F32(np.inf), F32(0), F32(1))) and ao.fma(F32(1e30), F32(1e30), F32(1)) == np.inf
    assert ao.fma(F32(2), F32(3), F32(-np.inf)) == -np.inf


@pytest.mark.parametrize("weight_decay", [0.0, 1e-4])
def test_oracle_against_torch_cpu_adam(weight_decay):
    """20 steps of torch.optim.Adam(foreach=False) on CPU tensors.  This comparison is a BOUND, not torch.equal: ATen's
    CPU kernels are vectorised without the FMAs its CUDA kernels contract to and its CPU addcmul multiplies
    (value * g) * g where the CUDA one multiplies value * (g * g).  Here exp_avg comes out equal and exp_avg_sq one
    ulp off in about a quarter of the elements per step, so the oracle, which restates the CUDA sequence, differs from
    them in the last bits, and both moments are recursions that carry the difference on.  Held after step t: exp_avg
    and exp_avg_sq within t + 1 ulps (plus 8 units of the smallest subnormal), the parameter within the accumulated
    rounding of its updates (an update is at most a few lr: 8 ulps of 10 lr plus one ulp of p per step)."""
    n = 4096
    torch.manual_seed(1)
    tp = torch.nn.Parameter(torch.randn(n))
    opt = torch.optim.Adam([tp], lr=1e-3, weight_decay=weight_decay, foreach=False)
    P, M, V = tp.detach().numpy().copy(), np.zeros(n, F32), np.zeros(n, F32)
    lr = 1e-3
    for step in range(1, 21):
        g = torch.randn(n)
        g[0], g[1], g[2], g[3], g[4] = 0.0, 1e-30, 1e30, -1e-30, 3e-21     # g[4]: v stays subnormal
        if step == 10:
            lr = 3e-4
            for group in opt.param_groups:
                group["lr"] = lr
        tp.grad = g.clone()
        opt.step()
        P, M, V = ao.adam_step(P, g.numpy(), M, V, lr=lr, weight_decay=weight_decay, step=step)
        st = opt.state[tp]
        tm, tv, tpn = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy(), tp.detach().numpy()
        assert np.array_equal(np.isfinite(tv), np.isfinite(V)) and np.isinf(V[2]) and np.all(np.isfinite(P))
        f = np.isfinite(V)
        assert np.all(np.abs(tm - M) <= (step + 1) * np.spacing(np.abs(M)))
        assert np.all(np.abs(tv[f] - V[f]) <= (step + 1) * np.spacing(np.abs(V[f])) + 8 * np.finfo(F32).smallest_subnormal)
        assert np.all(np.abs(tpn - P) <= step * (np.spacing(np.abs(P)) + 8 * 2.0 ** -24 * 10 * 1e-3))
    assert weight_decay != 0 or 0 < V[4] < np.finfo(F32).tiny    # with decay, wd * p dominates that gradient


def test_oracle_lerp_branches_and_specials():
    g = np.array([1.0, -2.0, 0.0, np.inf, np.nan, -0.0], F32)
    z = np.zeros(6, F32)
    for beta1 in (0.9, 0.3):                              # weight 0.1: self + w*(end - self); 0.7: the other form
        p, m, v = ao.adam_step(z, g, z, z, betas=(beta1, 0.999), step=1)
        assert np.allclose(m[:3], (1 - beta1) * g[:3], rtol=1e-6)
        assert np.isnan(p[3]) and np.isnan(p[4]) and np.isinf(v[3]) and np.isnan(m[4])
        assert p[2] == 0 and p[5] == 0 and m[2] == 0 and v[2] == 0
        assert np.allclose(p[:2], [-1e-3, 1e-3], rtol=1e-5)


# ------------------------------------------------------------------ the optimizer's state and checkpoints

def _module():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 4, 3), torch.nn.BatchNorm2d(4), torch.nn.Conv2d(4, 2, 1))


def _torch_steps(net, opt, n):
    for i in range(n):
        torch.manual_seed(100 + i)
        for p in net.parameters():
            p.grad = torch.randn_like(p)
        opt.step()


def test_constructor_matches_torch_defaults():
    net = _module()
    ours, theirs = optim.Adam(net.parameters()), torch.optim.Adam(net.parameters())
    for key in ("lr", "betas", "eps", "weight_decay"):
        assert ours.param_groups[0][key] == theirs.param_groups[0][key]
    assert set(ours.param_groups[0]) == {"params", "lr", "betas", "eps", "weight_decay"}
    assert ours.state_dict()["state"] == {}


def test_state_dict_round_trip_with_torch_adam(tmp_path):
    """torch.optim.Adam -> save_model -> pvnet_b200.optim.Adam -> save_model -> torch.optim.Adam, continued, equals an
    uninterrupted torch run: nothing in the state is lost or converted on the way."""
    straight = _module()
    opt_s = torch.optim.Adam(straight.parameters(), lr=2e-3, weight_decay=1e-4)
    _torch_steps(straight, opt_s, 3)

    a = _module()
    opt_a = torch.optim.Adam(a.parameters(), lr=2e-3, weight_decay=1e-4)
    _torch_steps(a, opt_a, 2)
    net_utils.save_model(a, opt_a, 4, str(tmp_path / "one"))

    b = _module()
    ours = optim.Adam(b.parameters(), lr=5.0)
    assert net_utils.load_model(b, ours, str(tmp_path / "one")) == 5
    assert ours.param_groups[0]["lr"] == 2e-3 and ours.param_groups[0]["weight_decay"] == 1e-4
    for p, q in zip(b.parameters(), a.parameters()):
        s, t = ours.state[p], opt_a.state[q]
        assert set(s) == {"step", "exp_avg", "exp_avg_sq"}
        assert s["step"].dtype == torch.float32 and s["step"].device.type == "cpu" and s["step"].dim() == 0
        assert float(s["step"]) == 2.0
        for key in ("exp_avg", "exp_avg_sq"):
            assert s[key].dtype == torch.float32 and s[key].stride() == p.stride() and torch.equal(s[key], t[key])
    assert ours.state_dict()["state"].keys() == opt_a.state_dict()["state"].keys()
    net_utils.save_model(b, ours, 5, str(tmp_path / "two"))

    c = _module()
    opt_c = torch.optim.Adam(c.parameters())
    assert net_utils.load_model(c, opt_c, str(tmp_path / "two")) == 6
    torch.manual_seed(102)                                # the third step's gradients
    for p in c.parameters():
        p.grad = torch.randn_like(p)
    opt_c.step()
    for p, q in zip(c.parameters(), straight.parameters()):
        assert torch.equal(p, q)
        assert torch.equal(opt_c.state[p]["exp_avg_sq"], opt_s.state[q]["exp_avg_sq"])
        assert float(opt_c.state[p]["step"]) == 3.0


def test_fresh_state_dict_loads_into_torch_adam():
    """A pvnet_b200.optim.Adam that has never stepped: its groups carry no torch-only keys, and torch fills them in."""
    net = _module()
    ours = optim.Adam(net.parameters(), lr=3e-3, betas=(0.8, 0.99), eps=1e-7, weight_decay=1e-5)
    theirs = torch.optim.Adam(net.parameters())
    theirs.load_state_dict(ours.state_dict())
    g = theirs.param_groups[0]
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"]) == (3e-3, (0.8, 0.99), 1e-7, 1e-5)
    assert g["amsgrad"] is False and g["maximize"] is False
    _torch_steps(net, theirs, 1)                          # and it steps


# ------------------------------------------------------------------ what a step passes down

class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, dev, tensors, lr, beta1, beta2, eps, weight_decay, step):
        self.calls.append({"n": len(tensors), "lr": lr, "betas": (beta1, beta2), "eps": eps,
                           "weight_decay": weight_decay, "step": step,
                           "params": [p for p, _, _, _ in tensors]})


@pytest.fixture
def recorded(monkeypatch):
    """optim.Adam.step with the native call replaced by a recorder and the device check lifted, so its host logic
    runs on CPU tensors."""
    rec = _Recorder()
    monkeypatch.setattr(optim, "_adam_step", rec)
    monkeypatch.setattr(optim, "_check_device", lambda p: None)
    return rec


def _set_grads(net):
    for p in net.parameters():
        p.grad = torch.ones_like(p)


def test_learning_rate_helpers_reach_the_native_call(recorded, capsys):
    net = _module()
    opt = optim.Adam(net.parameters(), lr=1e-3, weight_decay=1e-4)
    _set_grads(net)
    opt.step()
    net_utils.adjust_learning_rate(opt, 0, 0.5, 1)
    opt.step()
    net_utils.set_learning_rate(opt, 7e-4)
    opt.step()
    assert [c["lr"] for c in recorded.calls] == [1e-3, 5e-4, 7e-4]
    assert [c["step"] for c in recorded.calls] == [1, 2, 3]
    n = len(list(net.parameters()))
    assert all(c["n"] == n and c["betas"] == (0.9, 0.999) and c["eps"] == 1e-8 and c["weight_decay"] == 1e-4
               for c in recorded.calls)


def test_step_groups_by_step_value_and_skips_missing_gradients(recorded):
    net = _module()
    params = list(net.parameters())
    opt = optim.Adam(params)
    _set_grads(net)
    params[1].grad = None
    opt.step()
    assert recorded.calls[0]["n"] == len(params) - 1 and params[1] not in opt.state
    _set_grads(net)
    opt.step()                                            # params[1] reaches step 1, the others step 2
    second = recorded.calls[1:]
    assert sorted(c["step"] for c in second) == [1, 2]
    one = next(c for c in second if c["step"] == 1)
    assert one["n"] == 1 and one["params"][0] is params[1]
    assert float(opt.state[params[1]]["step"]) == 1.0 and float(opt.state[params[0]]["step"]) == 2.0


def test_param_groups_have_their_own_scalars(recorded):
    net = _module()
    opt = optim.Adam([{"params": net[0].parameters(), "lr": 1e-2},
                      {"params": net[2].parameters(), "weight_decay": 0.1}], lr=1e-3)
    _set_grads(net)
    assert opt.step(lambda: torch.tensor(3.0)) == 3.0
    assert [(c["lr"], c["weight_decay"], c["n"]) for c in recorded.calls] == [(1e-2, 0, 2), (1e-3, 0.1, 2)]


# ------------------------------------------------------------------ refusals

@pytest.mark.parametrize("option", ["amsgrad", "maximize", "foreach", "capturable", "differentiable", "fused"])
def test_torch_only_keywords_are_refused(option):
    for value in (True, False):
        with pytest.raises(ValueError, match=option):
            optim.Adam(_module().parameters(), **{option: value})


@pytest.mark.parametrize("kwargs", [{"lr": -1.0}, {"lr": float("nan")}, {"eps": -1e-8}, {"betas": (1.0, 0.999)},
                                    {"betas": (0.9, -0.1)}, {"weight_decay": -1.0}, {"lr": float("inf")}])
def test_bad_hyper_parameters_are_refused(kwargs):
    with pytest.raises(ValueError, match="Invalid"):
        optim.Adam(_module().parameters(), **kwargs)


def test_cpu_parameter_is_refused():
    net = _module()
    opt = optim.Adam(net.parameters())
    _set_grads(net)
    with pytest.raises(RuntimeError, match="runs only on CUDA"):
        opt.step()
    assert len(opt.state) == 0                            # nothing was created or advanced


def test_step_refusals_come_before_any_launch(recorded):
    def fresh(**kw):
        net = _module()
        _set_grads(net)
        return net, optim.Adam(net.parameters(), **kw)

    net, opt = fresh()
    net[0].weight.grad = torch.ones_like(net[0].weight).to_sparse()
    with pytest.raises(ValueError, match="sparse"):
        opt.step()

    net, opt = fresh()
    net[2].bias.data = net[2].bias.data.double()
    net[2].bias.grad = torch.ones(2, dtype=torch.float64)
    with pytest.raises(ValueError, match="float32"):
        opt.step()

    # a gradient laid out differently from its parameter is refused, not copied: channels_last against contiguous
    net, opt = fresh()
    net[0].weight.grad = torch.ones(4, 3, 3, 3).contiguous(memory_format=torch.channels_last)
    with pytest.raises(ValueError, match="strides"):
        opt.step()
    # the same layout on both sides is fine
    net, opt = fresh()
    net[0].weight.data = net[0].weight.data.contiguous(memory_format=torch.channels_last)
    net[0].weight.grad = torch.ones(4, 3, 3, 3).contiguous(memory_format=torch.channels_last)
    opt.step()
    assert opt.state[net[0].weight]["exp_avg"].stride() == net[0].weight.stride()

    # a parameter with gaps in memory
    base = torch.zeros(4, 8)
    p = torch.nn.Parameter(base[:, :4])
    p.grad = torch.ones(4, 8)[:, :4]
    with pytest.raises(ValueError, match="not dense"):
        optim.Adam([p]).step()

    # state of the wrong layout (loaded from elsewhere)
    net, opt = fresh()
    opt.step()
    opt.state[net[0].weight]["exp_avg"] = torch.zeros(4, 3, 3, 3).contiguous(memory_format=torch.channels_last)
    with pytest.raises(ValueError, match="exp_avg"):
        opt.step()

    # options a loaded torch state_dict may carry
    net, opt = fresh()
    src = torch.optim.Adam(net.parameters(), amsgrad=True)
    opt.load_state_dict(src.state_dict())
    with pytest.raises(ValueError, match="amsgrad"):
        opt.step()

    # every refusal above left the launch recorder with the two accepted steps only, and advanced no step count
    assert len(recorded.calls) == 2


def test_refused_step_advances_nothing(recorded):
    net = _module()
    opt = optim.Adam(net.parameters())
    _set_grads(net)
    opt.step()
    net[2].weight.grad = net[2].weight.grad.to_sparse()  # the last group member is refused
    with pytest.raises(ValueError):
        opt.step()
    assert all(float(opt.state[p]["step"]) == 1.0 for p in net.parameters()) and len(recorded.calls) == 1


# ------------------------------------------------------------------ the C ABI's checks (host side, no device needed)

def _call(tensors, n=None, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=1):
    table = (_native.AdamTensor * max(len(tensors), 1))(*(_native.AdamTensor(*t) for t in tensors))
    return _native.lib().pvnet_adam_step(table, len(tensors) if n is None else n, lr, beta1, beta2, eps, weight_decay,
                                         step, None)


def test_abi_refusals_and_no_ops():
    L = _native.lib()
    ok = (256, 512, 768, 1024, 16)                        # plausible aligned addresses: never dereferenced on the host
    cases = [
        (dict(n=-1), b"n_tensors"),
        (dict(step=0), b"step"),
        (dict(lr=-1e-3), b"lr"), (dict(lr=float("nan")), b"lr"), (dict(lr=float("inf")), b"lr"),
        (dict(eps=-1.0), b"eps"), (dict(weight_decay=float("inf")), b"weight_decay"),
        (dict(beta1=1.0), b"betas"), (dict(beta2=-0.5), b"betas"), (dict(beta1=float("nan")), b"betas"),
    ]
    for kw, word in cases:
        assert _call([ok], **kw) == -1, kw
        assert word in L.pvnet_last_error(), (kw, L.pvnet_last_error())
    assert L.pvnet_adam_step(None, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None) == -1
    assert b"null" in L.pvnet_last_error()
    for bad, word in (((256, 512, 768, 1024, -1), b"negative numel"), ((0, 512, 768, 1024, 4), b"null pointer"),
                      ((256, None, 768, 1024, 4), b"null pointer"), ((256, 512, 770, 1024, 4), b"4-byte"),
                      ((257, 512, 768, 1024, 4), b"4-byte")):
        assert _call([ok, bad]) == -1, bad
        assert word in L.pvnet_last_error() and b"tensor 1" in L.pvnet_last_error()
    # nothing to do: an empty table, and entries with numel == 0 whatever their pointers
    assert L.pvnet_adam_step(None, 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None) == 0
    before = _native.launch_count()
    assert _call([(None, None, None, None, 0), (3, 5, 7, 9, 0)]) == 0
    assert _native.launch_count() == before
    assert L.pvnet_adam_chunk_tensors() >= 77             # Resnet18_8s's parameter set is one launch
