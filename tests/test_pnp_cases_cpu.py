"""CPU: the uncertainty-PnP cases of tests/pnp_cases.py are what the GPU tests assume them to be.

The fp64 oracle's P3P recovers the generating pose to 1e-6 from the exact projections of every noise-free pn == 4
image but the listed ill-conditioned ones; the weights built to reorder the P3P points have the keys the GPU tests
rely on."""
import numpy as np
import pytest

from oracle import pnp_oracle as pn
from tests import pnp_cases as pc


@pytest.mark.parametrize("name", [n for n, _ in pc.P3P_BATCHES])
def test_oracle_p3p_recovers_the_generating_pose(name):
    c = pc.p3p_batch(name)
    uv = pc.project(c["P"], c["R"], c["t"], c["K"])
    z = np.einsum("nij,pj->npi", c["R"], c["P"].astype(np.float64))[..., 2] + c["t"][:, 2:]
    assert (z > 0.1 * c["unit"]).all()
    listed = set(pc.ORACLE_ILL_CONDITIONED.get(name, ()))
    missed, stale = [], []
    for i in range(pc.P3P_BATCH):
        got = pc.oracle_p3p(uv[i], c["w"][i], c["P"], c["K"])
        err = np.inf if got is None else pc.pose_error(got, c["R"][i], c["t"][i], c["unit"])
        if err > 1e-6 and i not in listed:
            missed.append((i, err))
        if err <= 1e-6 and i in listed:
            stale.append((i, err))                    # listed, but well-conditioned: it would escape the GPU bar
    assert not missed, missed
    assert not stale, stale
    assert len(listed) < 0.02 * pc.P3P_BATCH


def test_p3p_batches_reorder_the_points():
    c = pc.p3p_batch("cloud_a")
    keys = c["w"][..., 0].astype(np.float64) + c["w"][..., 1]
    assert all(len(set(k)) == 4 for k in keys)
    firsts = {int(np.argsort(k, kind="stable")[0]) for k in keys}
    assert firsts == {0, 1, 2, 3}                     # every point is left out of the solving three somewhere


def test_negative_key_and_filtered_weights():
    w = pn.covariance_to_weights(pc.cov_from_weight(pc.W_NEGATIVE_KEY)[None])[0]
    assert np.allclose(w, [1.0, -2.0, 5.0], rtol=1e-5) and w[0] + w[1] < 0
    for name, cov in pc.FILTERED_COVS.items():
        assert np.array_equal(pn.covariance_to_weights(cov[None]), np.zeros((1, 3))), name


@pytest.mark.parametrize("pn_", sorted(pc.POINT_COUNTS))
def test_noisy_problems_are_in_front_of_the_camera(pn_):
    c = pc.noisy_problems(f"count/{pn_}", pn_, 32, pc.POINT_COUNTS[pn_])
    assert c["kp"].shape == (32, pn_, 2) and np.isfinite(c["kp"]).all()
    z = np.einsum("nij,pj->npi", c["R"], c["P"].astype(np.float64))[..., 2] + c["t"][:, 2:]
    assert (z > 0.1 * c["unit"]).all()
    assert (np.linalg.eigvalsh(c["cov"].astype(np.float64)) > 0).all()
