"""Every device and pinned host allocation of the library is released by its owner: the handle's problem, layout and
dense-plan buffers by a re-layout or ``close``, a stand-alone call's buffers when it returns. Checked through
``b200ba_debug_live_allocations`` (count and bytes of everything the library holds)."""
import gc

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, synthetic

DENSE_MODES = ["own", "lib"]


def live():
    gc.collect()  # handles of earlier tests that nothing references any more are closed first
    return api.debug_live_allocations()


def small_problem():
    return synthetic.make_problem(2, n_imagesets=10, lattice=(10, 8), image_size=(410, 290))


def set_dense_mode(monkeypatch, mode):
    if mode == "lib":
        monkeypatch.setenv("B200BA_DENSE", "lib")
    else:
        monkeypatch.delenv("B200BA_DENSE", raising=False)


def held_by_fresh_handle(sp, eliminate_points):
    """What a new handle holds after one LM iteration at the layout of `eliminate_points`."""
    start = live()
    adj = api.BundleAdjuster(sp.problem, 0)
    adj.set_state(sp.init_state.copy())
    adj.optimize(cabi.default_options(max_iteration_count=1, eliminate_points=int(eliminate_points)))
    now = live()
    adj.close()
    assert live() == start
    return tuple(a - b for a, b in zip(now, start))


@pytest.mark.gpu
@pytest.mark.parametrize("dense", DENSE_MODES)
def test_handle_releases_everything_on_close(monkeypatch, dense):
    set_dense_mode(monkeypatch, dense)
    sp = small_problem()
    start = live()
    adj = api.BundleAdjuster(sp.problem, 0)
    assert live()[0] > start[0]
    adj.set_state(sp.init_state.copy())
    adj.optimize(cabi.default_options(max_iteration_count=2))
    adj.calibration_report(with_errors=True)
    adj.report_images(0)
    adj.delete_outliers(0, 6.0, np.ones(sp.problem.n_imagesets, bool))
    adj.snapshot_state()
    adj.restore_state()
    adj.run_bundle_adjustment(cabi.default_options(), 2, 1e-4)
    held = live()
    # the lazily created buffers are made once: a second round allocates nothing
    adj.calibration_report()
    adj.report_images(0)
    adj.snapshot_state()
    adj.run_bundle_adjustment(cabi.default_options(), 1, 1e-4)
    assert live() == held
    adj.close()
    assert live() == start


@pytest.mark.gpu
@pytest.mark.parametrize("dense", DENSE_MODES)
def test_relayout_holds_what_a_fresh_handle_holds(monkeypatch, dense):
    set_dense_mode(monkeypatch, dense)
    sp = small_problem()
    fresh = {e: held_by_fresh_handle(sp, e) for e in (True, False)}
    assert fresh[True] != fresh[False]
    start = live()
    adj = api.BundleAdjuster(sp.problem, 0)
    adj.set_state(sp.init_state.copy())
    for _ in range(3):
        for e in (True, False):
            adj.optimize(cabi.default_options(max_iteration_count=1, eliminate_points=int(e)))
            assert tuple(a - b for a, b in zip(live(), start)) == fresh[e]
    adj.close()
    assert live() == start


@pytest.mark.gpu
def test_stand_alone_calls_release_their_buffers():
    rng = np.random.default_rng(5)
    start = live()

    n = 300
    a = rng.standard_normal((n, n))
    api.dense_cholesky_solve(a @ a.T + n * np.eye(n), rng.standard_normal(n), block_width=128)
    assert live() == start

    bs, nb, nd = 3, 20, 12
    d = np.stack([np.eye(bs) * 4 + 0.1 * (m + m.T) for m in rng.standard_normal((nb, bs, bs))])
    b = 0.1 * rng.standard_normal((nb * bs, nd))
    api.schur_solve(bs, d, b, np.eye(nd) * 5, rng.standard_normal(nb * bs), rng.standard_normal(nd))
    assert live() == start

    w, h = 64, 48
    model = api.CentralGenericModel(6, 5, 0, 0, w - 1, h - 1, w, h)
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dirs = np.stack([(xs - w / 2) / 40.0, (ys - h / 2) / 40.0, np.ones_like(xs)], -1)
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    assert model.FitToDenseModel(dirs, 2, 3)
    model.FitToPixelDirections(np.stack([xs.ravel(), ys.ravel()], -1), dirs.reshape(-1, 3), 3)
    assert live() == start

    sites = rng.integers(0, 4 * np.array([w, h]), (50, 2))
    api.RenderVoronoi(w, h, sites, rng.uniform(0, 255, (50, 3)).astype(np.float32))
    assert live() == start
