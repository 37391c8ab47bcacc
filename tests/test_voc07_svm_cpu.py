"""CPU tests of the VOC07 linear-SVM evaluation: the fixture against the regenerated features, the restatements of
StratifiedKFold and average_precision_score against sklearn (when installed), the float64 oracle against sklearn's
LinearSVC, and a dry run of the solver's launch schedule against the C-ABI prototypes."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import voc07_oracle as V


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, V.GOLDEN))


def test_fixture_matches_the_regenerated_features(golden):
    xtr, ttr, xte, tte = V.synthetic_voc07()
    assert V.feature_digest(xtr, xte) == golden["features_sha256"]
    assert xtr.shape == (5011, 2048) and xte.shape == (4952, 2048) and ttr.shape == (5011, 20)
    assert (xtr >= 0).all() and np.allclose(np.linalg.norm(xtr, axis=1), 1, atol=1e-6)
    assert (ttr == -1).any() and (tte == -1).any() and ((ttr == 1).sum(1) > 1).any()
    _, fold, _ = V.problems(ttr)
    assert np.array_equal(fold, golden["fold_ids"].numpy())
    assert len(set(golden["oracle_best_cost"].tolist())) >= 2
    # the float64 optimum scores like the reference's sklearn run
    assert abs(golden["oracle_mean_ap"] - golden["ref_mean_ap"]) <= 2e-4
    assert np.abs(golden["oracle_cv_ap"].numpy() - golden["ref_cv_ap"].numpy()).max() <= 1e-3


@pytest.fixture(scope="module")
def small():
    return V.synthetic_voc07(n_train=400, n_test=300, dim=48, classes=4, seed=11)


def test_fold_restatement_equals_stratified_kfold(small):
    model_selection = pytest.importorskip("sklearn.model_selection")
    _, ttr, _, _ = small
    rng = np.random.default_rng(0)
    for y in [np.where(ttr[:, k] == 1, 1, -1) for k in range(ttr.shape[1])] + [rng.integers(0, 3, 101)]:
        for n_splits in (2, 3, 5):
            want = np.empty(len(y), int)
            for f, (_, test) in enumerate(model_selection.StratifiedKFold(n_splits).split(np.zeros(len(y)), y)):
                want[test] = f
            assert np.array_equal(V.stratified_folds(y, n_splits), want)


def test_ap_restatement_equals_sklearn():
    metrics = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(1)
    for n in (1, 2, 17, 1000):
        for ties in (False, True):
            s = rng.standard_normal(n)
            if ties:
                s = np.round(s * 2) / 2
            t = rng.integers(-1, 2, n)
            t[0] = 1
            keep = t != -1                       # difficult entries are excluded, as clf_voc07.py:96-104 does
            got = V.average_precision(t[keep] == 1, s[keep])
            assert abs(got - metrics.average_precision_score(t[keep] == 1, s[keep])) <= 1e-12


def test_oracle_objective_is_at_most_sklearns(small):
    svm = pytest.importorskip("sklearn.svm")
    xtr, ttr, _, _ = small
    _, _, cy = V.problems(ttr)
    xa = V.augment(xtr)
    W, _ = V.newton_cg(xa, cy)
    f = V.objective(xa, cy, W)
    y = np.where(ttr == 1, 1, -1)
    F = V.FOLDS + 1
    for k in range(ttr.shape[1]):
        for ci, cost in enumerate(V.SVM_COSTS):
            p = (k * len(V.SVM_COSTS) + ci) * F + V.FOLDS                # the full fit
            clf = svm.LinearSVC(C=cost, class_weight={1: 2, -1: 1}, penalty="l2", loss="squared_hinge",
                                max_iter=2000).fit(xtr, y[:, k])
            w = np.r_[clf.coef_[0], clf.intercept_]
            assert f[p] <= V.objective(xa, cy[:, p:p + 1], w[:, None])[0] * (1 + 1e-12)


# ---------------------------------------------------------------------------------------------------------- dry run
class _Event:
    def record(self):
        pass

    def query(self):
        return True


def test_solver_schedule_dry_run(monkeypatch):
    """The solver's launches against the prototypes and limits, on CPU tensors with a scripted device: two Newton
    steps of three CG iterations each.  The only host synchronisation is the one read per Newton step."""
    from virtex_b200 import ops, svm
    calls = []
    script = {"newton": [320, 320, 0], "cg": [2, 1, 0]}

    def put(ptr, v):
        ctypes.c_int32.from_address(ptr).value = v

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), name
        calls.append(name)
        if name == "vtx_svm_newton_begin":
            put(args[7], script["newton"].pop(0))
            script["cg_it"] = 0
        elif name == "vtx_svm_cg_scalars":
            put(args[5], script["cg"][script["cg_it"]])
            script["cg_it"] += 1

    def fake_gemm(A, B, D, M, N, K, a_mn=0, b_mn=0, tile_n=0, **kw):
        assert not kw and b_mn == 1 and D.dtype == torch.float32 and D.shape == (M, N)
        assert A.dtype == B.dtype == torch.bfloat16 and K % 64 == 0 and N % 64 == 0 and M % 64 == 0
        assert A.shape == ((M, K) if a_mn == 0 else (K, M)) and B.shape == (K, N)
        calls.append(("gemm", M, N, K, a_mn))

    syncs = []
    real_item = torch.Tensor.item
    monkeypatch.setattr(ops, "call", fake_call)
    monkeypatch.setattr(ops, "gemm", fake_gemm)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(svm, "_pinned_counts", lambda n: torch.zeros(n, dtype=torch.int32))
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.Tensor, "item", lambda t: syncs.append(len(calls)) or real_item(t))
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: pytest.fail("synchronize"))

    n, d, nt, P = 5011, 2048, 4952, 320
    cy = torch.zeros(5056, P)
    out = svm._solve(torch.zeros(n, d), torch.zeros(nt, d), cy, 2112, P)
    assert out["z"].shape == (5056, P) and out["z_test"].shape == (4992, P) and out["w"].shape == (2112, P)
    newton = ["gemm", "vtx_svm_margin", "gemm", "vtx_svm_axpy_dot", "vtx_svm_newton_begin"]
    cg = ["gemm", "vtx_svm_hess_mid", "gemm", "vtx_svm_axpy_dot", "vtx_svm_cg_update", "vtx_svm_cg_scalars",
          "vtx_svm_cg_direction"]
    step = ["vtx_svm_split_cols", "gemm", "vtx_svm_axpy_dot", "vtx_svm_line_search", "vtx_svm_newton_step"]
    names = [c[0] if isinstance(c, tuple) else c for c in calls]
    want = (["vtx_svm_split_x"] + (newton + ["vtx_svm_cg_start"] + 3 * cg + step) * 2 + newton
            + ["vtx_svm_split_x", "gemm"])
    assert names == want
    # one read per Newton step, each right after vtx_svm_newton_begin
    assert len(syncs) == 3 and all(names[i - 1] == "vtx_svm_newton_begin" for i in syncs)
    gemms = {c[1:] for c in calls if isinstance(c, tuple)}
    assert gemms == {(5056, P, 3 * 2112, 0), (2112, P, 3 * 5056, 1), (4992, P, 3 * 2112, 0)}


def test_solver_limits_are_the_kernels():
    """The padded sizes the solver accepts stay inside the kernels' shared-memory staging (include/virtex_b200.h)."""
    from virtex_b200 import svm
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "virtex_b200.h")).read()
    assert "#define VTX_SVM_MAX_N 16384" in header and "#define VTX_SVM_SLICES 32" in header
    assert "#define VTX_SVM_NSCAL 7" in header and "#define VTX_SVM_NFLAGS 6" in header
    with pytest.raises(ValueError, match="16384"):
        svm.train_test_svms(np.zeros((16385, 4), np.float32), np.ones((16385, 1)), np.zeros((2, 4), np.float32),
                            np.ones((2, 1)))
