"""ovp_transfer_bytes counts every host<->device copy an entry point issues: for each call below the two counters grow by exactly the bytes of
its host operands and results, plus the state column indices it uploads (4 bytes each) and the two device status words an update reads
back (8 bytes)."""
import numpy as np
import pytest

import update_reference as ur
from ov_plane_b200 import api

pytestmark = pytest.mark.gpu

N_CLONES = 4
STATUS_WORDS = 8


@pytest.fixture(scope="module")
def state():
    c = api.Context(ur.STATE_OPTIONS, device=0, max_state=128, max_meas_rows=1024)
    rng = np.random.default_rng(7)
    clones = []
    for k in range(N_CLONES):
        q = rng.standard_normal(4)
        q /= np.linalg.norm(q)
        pose = np.concatenate([q, rng.standard_normal(3)])
        clones.append(c.add_clone_raw(0.1 * (k + 1), pose, pose))
    imu = c.handle_imu()
    c.ekf_update([imu], rng.standard_normal((4, 15)), rng.standard_normal(4), np.ones(4))  # uploads the variable table once
    yield c, clones
    c.close()


def moved(ctx, call):
    h0, d0 = ctx.transfer_bytes()
    out = call()
    h1, d1 = ctx.transfer_bytes()
    return h1 - h0, d1 - d0, out


@pytest.mark.parametrize("with_R", [False, True])
def test_ekf_update(state, with_R):
    ctx, _ = state
    rows, n = 10, 15
    rng = np.random.default_rng(1)
    H, r = rng.standard_normal((rows, n)), 1e-3 * rng.standard_normal(rows)
    R = np.full(rows, 4.0) if with_R else None
    h2d, d2h, _ = moved(ctx, lambda: ctx.ekf_update([ctx.handle_imu()], H, r, R))
    assert h2d == 4 * n + 8 * rows * n + 8 * rows * (2 if with_R else 1)
    assert d2h == STATUS_WORDS


def test_get_marginal_covariance(state):
    ctx, clones = state
    hs = [ctx.handle_imu(), clones[0]]
    n = 15 + 6
    h2d, d2h, P = moved(ctx, lambda: ctx.get_marginal_covariance(hs))
    assert P.shape == (n, n)
    assert (h2d, d2h) == (4 * n, 8 * n * n)


@pytest.mark.parametrize("plane", [False, True])
def test_nullspace_project_inplace(state, plane):
    ctx, _ = state
    rows, hf, hx = 20, 3, 12
    rng = np.random.default_rng(2)
    Hf, Hx, r = rng.standard_normal((rows, hf)), rng.standard_normal((rows, hx)), rng.standard_normal(rows)
    Hcp = rng.standard_normal((rows, 3)) if plane else None
    ncp = 3 if plane else 0
    h2d, d2h, _ = moved(ctx, lambda: ctx.nullspace_project_inplace(Hf, Hx, r, Hcp))
    assert h2d == 8 * rows * (hf + hx + ncp + 1)
    assert d2h == 8 * (rows - hf) * (hx + ncp + 1)


@pytest.mark.parametrize("plane", [False, True])
def test_measurement_compress_inplace(state, plane):
    ctx, _ = state
    rows, cols = 40, 12
    rng = np.random.default_rng(3)
    Hx, r = rng.standard_normal((rows, cols)), rng.standard_normal(rows)
    Hcp = rng.standard_normal((rows, 3)) if plane else None
    ncp = 3 if plane else 0
    h2d, d2h, _ = moved(ctx, lambda: ctx.measurement_compress_inplace(Hx, r, Hcp))
    assert h2d == 8 * rows * (cols + ncp + 1)
    assert d2h == 8 * (cols + ncp + 1) * cols  # the leading columns of the Gram factor


def test_feature_jacobian_full(state):
    ctx, clones = state
    m = len(clones)
    rng = np.random.default_rng(4)
    uv = rng.uniform(-0.2, 0.2, (m, 2)).astype(np.float32)
    pf = np.array([0.3, -0.2, 4.0])
    h2d, d2h, (Hf, Hx, res, _) = moved(ctx, lambda: ctx.feature_jacobian_full(clones, uv, pf, pf, 0, None, None, 1.0, 1.0))
    rows = 2 * m
    assert Hf.shape == (rows, 3) and Hx.shape == (rows, 6 + 8 + 6 * m) and res.shape == (rows,)
    assert h2d == 4 * m + 8 * m  # clone handles, uv (float32 pairs)
    assert d2h == 8 * rows * (Hf.shape[1] + Hx.shape[1] + 1)
