"""GPU tests of the VOC07 linear-SVM evaluation (virtex_b200/svm.py, csrc/svm.cu) against the float64 oracle and the
reference's own sklearn run recorded in tests/golden/voc07_svm.pt."""
import os
import warnings

import numpy as np
import pytest
import torch

from tests import voc07_oracle as V

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, V.GOLDEN))


@pytest.fixture(scope="module")
def data():
    return V.synthetic_voc07()


@pytest.fixture(scope="module")
def solved(data):
    from virtex_b200.svm import SvmConvergenceWarning, train_test_svms
    xtr, ttr, xte, tte = data
    torch.cuda.set_device(0)
    with warnings.catch_warnings():
        warnings.simplefilter("error", SvmConvergenceWarning)   # every problem converges at the VOC07 shape
        return train_test_svms(torch.from_numpy(xtr).cuda(), ttr, torch.from_numpy(xte).cuda(), tte)


def _ap_gpu(scores, labels, folds, cols):
    from virtex_b200 import ops
    s = torch.from_numpy(scores).cuda()
    lab = torch.from_numpy(labels).cuda()
    fo = torch.from_numpy(folds).cuda()
    c = torch.from_numpy(np.asarray(cols, np.int32)).cuda()
    ap = torch.empty(len(cols), dtype=torch.float64, device="cuda")
    ops.call("vtx_svm_average_precision", s.data_ptr(), s.stride(0), s.shape[0], lab.data_ptr(), lab.stride(0),
             fo.data_ptr(), fo.stride(0), c.data_ptr(), len(cols), ap.data_ptr(), ops._stream())
    return ap.cpu().numpy()


@pytest.mark.parametrize("n", [1, 5011, 16384])
def test_average_precision_kernel_equals_restatement(n):
    rng = np.random.default_rng(n)
    C = 6
    scores = rng.standard_normal((n, C)).astype(np.float32)
    scores[:, 1] = np.round(scores[:, 1] * 4) / 4           # heavy ties
    scores[:, 2] = 0.5                                      # one threshold
    labels = (rng.random((n, C)) < 0.3).astype(np.int8)
    labels[rng.random((n, C)) < 0.1] = -1                   # excluded
    labels[:, 3] = 0                                        # no positive
    labels[0, 4] = 1
    folds = rng.integers(0, 3, (n, C)).astype(np.int8)
    cols = [(c, c, -1) for c in range(C)] + [(c, c, f) for c in (0, 1) for f in range(3)] + [(1, 0, 2)]
    got = _ap_gpu(scores, labels, folds, cols)
    for j, (sc, lc, f) in enumerate(cols):
        keep = (labels[:, lc] >= 0) & ((folds[:, lc] == f) if f >= 0 else True)
        want = V.average_precision(labels[keep, lc] == 1, scores[keep, sc].astype(np.float64))
        assert abs(got[j] - want) <= 1e-12, (n, j, got[j], want)


def test_average_precision_rejects_more_than_16384_samples():
    from virtex_b200.lib import VtxError
    n = 16385
    with pytest.raises(VtxError, match="16384"):
        _ap_gpu(np.zeros((n, 1), np.float32), np.zeros((n, 1), np.int8), np.zeros((n, 1), np.int8), [(0, 0, -1)])


def test_split_operand_products_match_float64(data):
    """The three-term products hi.hi + hi.lo + lo.hi of both shapes: each operand is split to ~2^-17 relative and the
    dropped lo.lo term is ~2^-18, so every output is within 2^-16 sum_k |a_k b_k| of the float64 product (fp32
    accumulation over K <= 15 168 adds less than 2^-24 K)."""
    from virtex_b200 import ops, svm
    xtr = torch.from_numpy(data[0]).cuda()
    n, d = xtr.shape
    n_pad, dp, P = 5056, 2112, 320
    xcat = torch.empty(n_pad, 3 * dp, dtype=torch.bfloat16, device="cuda")
    xstk = torch.empty(3 * n_pad, dp, dtype=torch.bfloat16, device="cuda")
    st = ops._stream()
    ops.call("vtx_svm_split_x", xtr.data_ptr(), d, n, d, n_pad, dp, xcat.data_ptr(), xstk.data_ptr(), st)
    g = torch.Generator().manual_seed(3)
    W = torch.zeros(dp, P)
    W[:d + 1] = torch.randn(d + 1, P, generator=g, dtype=torch.float64).float() * 3
    U = torch.zeros(n_pad, P)
    U[:n] = torch.randn(n, P, generator=g, dtype=torch.float64).float() * 20
    Wd, Ud = W.cuda(), U.cuda()
    wop = torch.empty(3 * dp, P, dtype=torch.bfloat16, device="cuda")
    uop = torch.empty(3 * n_pad, P, dtype=torch.bfloat16, device="cuda")
    ops.call("vtx_svm_split_cols", Wd.data_ptr(), dp, P, wop.data_ptr(), st)
    ops.call("vtx_svm_split_cols", Ud.data_ptr(), n_pad, P, uop.data_ptr(), st)
    Z = torch.empty(n_pad, P, device="cuda")
    G = torch.empty(dp, P, device="cuda")
    svm._gemm(xcat, wop, Z, n_pad, 3 * dp, 0)
    svm._gemm(xstk, uop, G, dp, 3 * n_pad, 1, tile_n=64)
    xa = np.zeros((n_pad, dp))
    xa[:n, :d + 1] = V.augment(data[0])
    Wn, Un = W.double().numpy(), U.double().numpy()
    for got, want, bound in ((Z, xa @ Wn, np.abs(xa) @ np.abs(Wn)), (G, xa.T @ Un, np.abs(xa).T @ np.abs(Un))):
        err = np.abs(got.cpu().double().numpy() - want)
        assert (err <= 2.0 ** -16 * bound + 1e-30).all(), float((err / (bound + 1e-30)).max())
    assert float(Z[n:].abs().max()) == 0.0


def test_every_problem_reaches_the_float64_optimum(data, golden, solved):
    xtr, ttr, _, _ = data
    _, _, cy = V.problems(ttr)
    K, nc, F = ttr.shape[1], len(V.SVM_COSTS), V.FOLDS + 1
    W = solved.weights.double().numpy().reshape(K * nc * F, -1).T
    f = V.objective(V.augment(xtr), cy, W)
    f_opt = golden["oracle_objective"].numpy()
    gap = f / f_opt - 1
    print(f"objective gap: max {gap.max():.2e}, median {np.median(gap):.2e}; Newton steps "
          f"{int(solved.newton_steps.min())}..{int(solved.newton_steps.max())}, CG iterations "
          f"{int(solved.cg_iterations.max())} (most in one problem)")
    assert (f <= f_opt * (1 + 1e-6)).all(), np.argsort(-gap)[:5]


def test_aps_match_the_oracle(golden, solved):
    cv = solved.cv_ap.numpy()
    te = solved.test_ap_all.numpy()
    assert np.abs(cv - golden["oracle_cv_ap"].numpy()).max() <= 1e-3
    assert np.abs(te - golden["oracle_test_ap_all"].numpy()).max() <= 1e-3
    assert abs(solved.mean_ap - golden["oracle_mean_ap"]) <= 2e-4
    assert abs(solved.mean_ap - golden["ref_mean_ap"]) <= 2e-4
    print(f"mAP {solved.mean_ap:.6f}, oracle {golden['oracle_mean_ap']:.6f}, reference {golden['ref_mean_ap']:.6f}")


def test_best_cost_matches_the_oracle_where_it_is_decided(golden, solved):
    means = golden["oracle_cv_ap"].numpy().mean(2)
    top2 = np.sort(means, 1)[:, -2:]
    decided = top2[:, 1] - top2[:, 0] > 1e-4
    assert decided.sum() >= 10
    got, want = solved.best_cost.numpy(), golden["oracle_best_cost"].numpy()
    assert (got[decided] == want[decided]).all()
    assert np.array_equal(solved.test_ap.numpy(), solved.test_ap_all.numpy()[
        np.arange(len(got)), [V.SVM_COSTS.index(c) for c in got]])
    assert torch.equal(solved.coef, solved.weights[torch.arange(len(got)), [V.SVM_COSTS.index(c) for c in got], -1, :-1])


def test_fold_ids_equal_the_fixture(data, golden):
    _, fold, _ = V.problems(data[1])
    assert np.array_equal(fold, golden["fold_ids"].numpy())


def test_two_calls_are_bit_identical(data, solved):
    from virtex_b200.svm import train_test_svms
    xtr, ttr, xte, tte = data
    again = train_test_svms(xtr, ttr, xte, tte)        # numpy input: moved to the GPU
    assert torch.equal(again.weights, solved.weights)
    assert torch.equal(again.cv_ap, solved.cv_ap) and torch.equal(again.test_ap_all, solved.test_ap_all)
    assert again.mean_ap == solved.mean_ap


def test_input_validation():
    from virtex_b200.svm import train_test_svms
    rng = np.random.default_rng(0)
    x = rng.random((60, 8)).astype(np.float32)
    t = (rng.random((60, 2)) < 0.5).astype(np.int32)
    bad = t.copy()
    bad[0, 0] = 2
    with pytest.raises(ValueError, match="present"):
        train_test_svms(x, bad, x, t)
    one = t.copy()
    one[:, 1] = 0
    with pytest.raises(ValueError, match="one label value"):
        train_test_svms(x, one, x, t)
    with pytest.raises(ValueError):
        train_test_svms(x, t, x[:, :4], t)
    with pytest.raises(ValueError):
        train_test_svms(x, t[:50], x, t)
    with pytest.raises(ValueError, match="16384"):
        train_test_svms(np.zeros((16385, 8), np.float32), np.ones((16385, 1)), x, t[:, :1])


def test_small_problem_matches_the_oracle():
    """A shape that pads every dimension (n, d + 1 and P not multiples of 64)."""
    from virtex_b200.svm import train_test_svms
    xtr, ttr, xte, tte = V.synthetic_voc07(n_train=301, n_test=257, dim=37, classes=3, seed=5)
    r = train_test_svms(xtr, ttr, xte, tte)
    _, _, cy = V.problems(ttr)
    W_opt, _ = V.newton_cg(V.augment(xtr), cy)
    xa = V.augment(xtr)
    f_opt = V.objective(xa, cy, W_opt)
    f = V.objective(xa, cy, r.weights.double().numpy().reshape(-1, 38).T)
    assert (f <= f_opt * (1 + 1e-6)).all()
    cv, te, best, test_ap = V.evaluate(W_opt, xtr, ttr, xte, tte)
    assert np.abs(r.cv_ap.numpy() - cv).max() <= 1e-3 and np.abs(r.test_ap_all.numpy() - te).max() <= 1e-3


def test_a_problem_at_the_newton_cap_warns(monkeypatch):
    from virtex_b200 import svm
    xtr, ttr, xte, tte = V.synthetic_voc07(n_train=301, n_test=257, dim=37, classes=3, seed=5)
    monkeypatch.setattr(svm, "MAX_NEWTON", 1)
    with pytest.warns(svm.SvmConvergenceWarning, match="Newton-step"):
        r = svm.train_test_svms(xtr, ttr, xte, tte)
    assert int(r.newton_steps.max()) == 1
