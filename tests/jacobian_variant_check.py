"""Checks of the residual / Jacobian kernel under one instantiation variant against the CPU oracle.

The variants (B200BA_JAC_MINB, B200BA_JAC_THREADS, B200BA_COMPACT_J) are read once per process, so each one
needs a process of its own: tests/test_model_edges.py starts this script with the variant's environment.
Runs the crafted central-generic problem of test_model_edges.py and a small config-4 rig (two central-generic
cameras) under evaluation budgets 16 and 3, compares residuals, Jacobians (intrinsics in global columns) and
H / b with the oracle, and prints one JSON line with the variant in effect, the worst value of every
quantity and the cases that failed."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KEYS = ("B200BA_JAC_MINB", "B200BA_JAC_THREADS", "B200BA_COMPACT_J")


def main():
    from camera_calibration_b200 import cabi, synthetic
    from oracle import oracle
    from tests import test_model_edges as tme
    oracle.build()
    rig = synthetic.make_problem(4, n_imagesets=10, lattice=(10, 8), image_size=(410, 290))
    tme._CRAFTED["config4_rig"] = (rig, None)
    worst, failed = {}, []
    for name in ("central", "config4_rig"):
        for budget in (16, 3):
            case = f"{name} budget={budget}"
            try:
                if name == "config4_rig":
                    w = run_plain(oracle, rig, budget)
                else:
                    w = tme.run_crafted(oracle, name, budget, lm=False)[0]
            except AssertionError as e:
                failed.append({"case": case, "error": str(e)[:300]})
                continue
            for k, v in w.items():
                worst[k] = max(worst.get(k, 0.0), v)
    variant = {k: os.environ[k] for k in KEYS if k in os.environ}
    print(json.dumps({"variant": variant, "worst": worst, "failed": failed}))


def run_plain(oracle, sp, budget):
    from camera_calibration_b200 import api, cabi
    from tests import test_model_edges as tme
    lib = tme._lib()
    opt = cabi.default_options()
    try:
        lib.b200ba_debug_set_eval_budget(budget)
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            g = adj.evaluate(opt, compute_jacobians=True)
            lastp = adj.get_state().last_projection
            adj.set_state(sp.init_state)
            H, b, c = adj.build_system(opt)
    finally:
        lib.b200ba_debug_set_eval_budget(16)
    w = tme.check_evaluation(g, lastp, oracle.evaluate(sp.problem, sp.init_state, opt, True))
    w.update(tme.check_system(H, b, c, *oracle.build_system(sp.problem, sp.init_state, opt)))
    return w


if __name__ == "__main__":
    main()
