"""Pins the CPU oracle (oracle/fcma_oracle.c, TEST INFRASTRUCTURE) against
 (1) the known-answer values hard-coded in the reference's own tests, and
 (2) outputs of the unmodified reference committed under tests/golden/ (make_golden.py)."""
import numpy as np
import pytest

from oracle import fcma_oracle as orc

# reference tests/fcma/test_voxel_selection.py:58-65 (golden within-subject normalisation block)
REF_EXPECTED_FAKE_CORR = np.array(
    [[[1.06988919, 0.51641309, -0.46790636, -1.31926763, 0.2270218],
      [-1.22142744, -1.39881694, -1.2979387, 1.05702305, -0.6525566],
      [0.89795232, 1.27406132, 0.36460185, 0.87538344, 1.5227468],
      [-0.74641371, -0.39165771, 1.40124381, -0.61313909, -1.0972116]]])


def test_normaliser_known_answer(golden):
    g = golden("vs_small")
    z = orc.within_subject_norm(g["fake_corr"].copy(), 4)
    assert np.allclose(z, REF_EXPECTED_FAKE_CORR)          # the reference test's own tolerance
    assert np.allclose(g["scipy_norm"], REF_EXPECTED_FAKE_CORR)
    # bit-level agreement with the compiled reference C++ on the same input
    assert np.array_equal(z, g["cpp_norm"])


@pytest.mark.parametrize("tag", ["", "2"])
def test_small_stages_vs_reference(golden, tag):
    g = golden("vs_small")
    raw = list(g["raw1" if tag else "raw"])
    raw2 = list(g["raw2"]) if tag else None
    r, z, K = orc.voxel_block(raw, raw2, 0, 5, 4)
    # the reference's sgemm is a sequential fp32 FMA chain: the restatement is bit-exact
    assert np.array_equal(r, g["corr_raw" + tag])
    assert np.array_equal(z, g["corr_norm" + tag])
    assert np.max(np.abs(K - g["kernels" + tag])) <= 2e-6 * np.max(np.abs(g["kernels" + tag]))
    # within-subject norm applied to the reference's own raw corr is bit-exact
    z_ref_in = orc.within_subject_norm(g["corr_raw" + tag].copy(), 4)
    assert np.array_equal(z_ref_in, g["corr_norm" + tag])
    if tag:   # two masks: no self-correlation column, everything is well conditioned
        assert np.max(np.abs(z - g["corr_norm2"])) <= 5e-5
        assert np.max(np.abs(K - g["kernels2"])) <= 1e-4 * np.max(np.abs(g["kernels2"]))


def test_mid_stages_vs_reference(golden):
    g = golden("vs_mid")
    s, nb = g["task"]
    eps = int(g["eps"])
    r = orc.corr_block(list(g["raw"]), None, int(s), int(nb))
    assert r.shape == g["corr_raw"].shape
    assert np.array_equal(r, g["corr_raw"])          # bit-exact, self-correlation column included
    z = orc.within_subject_norm(g["corr_raw"].copy(), eps)
    assert np.array_equal(z, g["corr_norm"])
    # trailing epochs (E=10, eps=4 -> epochs 8,9) are left untouched (fcma_extension.cc:52)
    assert np.array_equal(z[:, 8:, :], g["corr_raw"][:, 8:, :])
    K = orc.kernel_matrices(g["corr_norm"])
    for i in range(K.shape[0]):
        orc.shrink_(K[i])
    assert np.max(np.abs(K - g["kernels"])) <= 2e-6 * np.max(np.abs(g["kernels"]))
    # two masks, ragged block
    s2, nb2 = g["task2"]
    r2 = orc.corr_block(list(g["d1"]), list(g["d2"]), int(s2), int(nb2))
    assert np.array_equal(r2, g["corr_raw2"])
    z2 = orc.within_subject_norm(r2.copy(), 4)
    assert np.array_equal(z2, g["corr_norm2"])
    K2 = orc.kernel_matrices(z2)
    for i in range(K2.shape[0]):
        orc.shrink_(K2[i])
    assert np.max(np.abs(K2 - g["kernels2"])) <= 1e-5 * np.max(np.abs(g["kernels2"]))


def test_classifier_kernel_vs_reference(golden):
    g = golden("clf")
    x1, x2 = list(g["big_x1"]), list(g["big_x2"])
    K, nd = orc.classifier_kernel(x1, x2, int(g["big_eps"]), int(g["big_portion"]))
    assert nd == int(g["big_num_digits"])
    assert np.max(np.abs(K - g["big_kernel"])) <= 1e-5 * np.max(np.abs(g["big_kernel"]))
    d5 = list(g["d5"])
    K12, nd12 = orc.classifier_kernel(d5[:12], d5[:12], 4, 2000)
    assert nd12 == int(g["one_num_digits"])
    # bit-exact correlations -> the 5 self-correlation features carry the reference's own clamp noise
    assert np.max(np.abs(K12 - g["one_kernel12"])) <= 2e-6 * np.max(np.abs(K12))


def test_compute_correlation_vs_reference(golden):
    g = golden("util")
    assert np.allclose(orc.compute_correlation(g["mat1"], g["mat1"]), g["c11"], atol=1e-5)
    assert np.allclose(orc.compute_correlation(g["mat1"], g["mat2"]), g["c12"], atol=1e-5)
    # the reference test's own oracle: np.corrcoef (tests/fcma/test_util.py:29-39)
    assert np.allclose(g["c11"], np.corrcoef(g["mat1"]), atol=1e-5)
    assert np.allclose(orc.compute_correlation(g["big1"], g["big2"]), g["cb"], atol=1e-5)
    c0 = orc.compute_correlation(g["mat1n"], g["mat2n"], return_nans=False)
    assert np.all(c0[0] == 0) and np.sum(c0 == 0) == 6
    c1 = orc.compute_correlation(g["mat1n"], g["mat2n"], return_nans=True)
    assert np.all(np.isnan(c1[0])) and np.sum(np.isnan(c1)) == 6
    assert np.array_equal(np.isnan(c1), np.isnan(g["cn1"]))


def test_epoch_normalize_vs_reference_golden_file(golden):
    g = golden("preproc")
    # rebuild the epochs exactly as preprocessing.py:68-86 does, normalising with the oracle
    out = []
    for sid in range(g["epochs"].shape[0]):
        ep = g["epochs"][sid]
        for cond in range(ep.shape[0]):
            for eid in range(ep.shape[1]):
                if ep[cond, eid].sum() > 0:
                    mat = g["activity"][sid][:, ep[cond, eid] == 1]
                    out.append(orc.epoch_normalize(np.ascontiguousarray(mat.T)))
    exp = g["expected_raw_data"]     # the reference's own golden file
    assert len(out) == len(exp)
    for a, b in zip(out, exp):
        assert np.allclose(a, b)     # tolerance of test_preprocessing.py:38-40
    # synthetic case with a constant voxel and unequal epoch lengths
    k = 0
    for sid in range(g["ep2"].shape[0]):
        ep = g["ep2"][sid]
        for cond in range(ep.shape[0]):
            for eid in range(ep.shape[1]):
                if ep[cond, eid].sum() > 0:
                    mat = g["act2"][sid][:, ep[cond, eid] == 1]
                    got = orc.epoch_normalize(np.ascontiguousarray(mat.T))
                    ref = g["raw2_%d" % k]
                    # the constant voxel: scipy's float32 moments leave rounding residue there
                    # ("Precision loss" warning in the reference); exact math gives 0.
                    live = np.ones(got.shape[1], bool)
                    if sid == 1:
                        live[7] = False
                        assert np.all(got[:, 7] == 0)
                    assert np.allclose(got[:, live], ref[:, live], atol=2e-6)
                    assert np.allclose(orc.epoch_normalize_numpy(mat.T)[:, live], ref[:, live],
                                       atol=2e-6)
                    k += 1
    assert k == 12


def test_oracle_vs_reference_golden_one_mask_all_voxels(golden):
    """vs_sym fixture (unmodified reference, one mask, V = 560 > two 256-row tiles): the oracle reproduces the
    reference's shrunk kernels of every voxel; the normalised correlations are symmetric in (i, j) up to fp32
    rounding away from the self column -- the property the symmetric CUDA pipeline rests on."""
    g = golden("vs_sym")
    raw, eps = list(g["raw"]), int(g["eps"])
    V = raw[0].shape[1]
    for s0, nb in ((0, 64), (250, 70), (V - 40, 40)):
        _, z, K = orc.voxel_block(raw, None, s0, nb, eps, shrink=True)
        ref = g["kernels"][s0:s0 + nb]
        assert np.max(np.abs(K - ref)) <= 2e-6 * np.max(np.abs(ref))
    _, zA, _ = orc.voxel_block(raw, None, 0, 48, eps, shrink=False)          # rows 0..47
    _, zB, _ = orc.voxel_block(raw, None, 300, 48, eps, shrink=False)        # rows 300..347
    a = zA[:, :, 300:348]                                                    # z(i, :, j), i < 48, j in 300..347
    b = np.transpose(zB[:, :, 0:48], (2, 1, 0))                              # z(j, :, i) rearranged to [i, e, j]
    assert np.max(np.abs(a - b)) <= 5e-6


def _svm_problem(rng, E, T, sig, classes=2):
    lab = np.array([e % classes for e in range(E)])
    Z = rng.randn(E, T).astype(np.float32)
    for c in range(classes):
        Z[lab == c, 5 * c:5 * c + 5] += sig
    K = (Z @ Z.T).astype(np.float32)
    digits = len(str(int(K[0, 0])))
    if digits > 2:                                   # the decimal shrink of voxelselector.py:409-412
        K = (K * np.float32(10.0 ** (2 - digits))).astype(np.float32)
    return K, lab


@pytest.mark.parametrize("E,T,sig,C,tol", [(32, 200, 0.35, 1.0, 1e-3), (64, 60, 0.2, 1.0, 1e-3), (48, 20, 0.3, 1.0, 1e-3),
                                           (64, 30, 0.1, 100.0, 1e-3), (32, 200, 0.3, 0.05, 1e-4)])
def test_svm_solver_restatement_equals_scikit_learn(E, T, sig, C, tol):
    """a8 (voxelselector.py:41-53 -> scikit-learn's libsvm, a third-party dependency of the reference): the sequential
    restatement in oracle/svm_oracle.c -- the algorithm the CUDA solver k_svm_cv implements -- against
    SVC.fit on the same precomputed kernels: iteration count, support set, dual coefficients and offset are IDENTICAL, without
    and with the shrinking heuristic (which demonstrably acts on the longer problems: svm_last_stats)."""
    from sklearn import svm
    rng = np.random.RandomState(E + T)
    shrunk = 0
    for _ in range(8):
        K, lab = _svm_problem(rng, E, T, sig)
        tr = np.arange(E)[np.arange(E) % 4 != 0]
        pos = [int(i) for i in tr if lab[i] == 0]
        neg = [int(i) for i in tr if lab[i] == 1]
        its = {}
        for shrinking in (False, True):
            clf = svm.SVC(kernel="precomputed", C=C, tol=tol, shrinking=shrinking)
            clf.fit(K[np.ix_(tr, tr)].astype(np.float64), lab[tr])
            alpha, rho, it = orc.svm_smo(K, pos + neg, len(pos), C, tol, -1, shrinking)
            its[shrinking] = it
            min_active, reconstructs = orc.svm_last_stats()
            assert shrinking or (min_active == len(tr) and reconstructs == 0)
            shrunk += shrinking and min_active < len(tr) and reconstructs > 0
            assert it == int(np.asarray(clf.n_iter_).ravel()[0])
            coef = alpha * np.r_[np.ones(len(pos)), -np.ones(len(neg))]
            mine = {i: coef[k] for k, i in enumerate(pos + neg) if alpha[k] != 0}
            sv = [int(i) for i in tr[clf.support_]]
            assert sorted(mine) == sorted(sv)
            # scikit-learn flips the signs of a two-class model (classes_[1] is the positive side of decision_function)
            assert all(mine[i] == -clf.dual_coef_[0][k] for k, i in enumerate(sv))
            assert rho == clf.intercept_[0]
    if T < 200:          # the problems of several hundred iterations: variables were shrunk and the gradient reconstructed
        assert shrunk >= 4


@pytest.mark.parametrize("classes,folds", [(2, 4), (3, 3), (4, 3)])
def test_svm_cross_validation_restatement_equals_scikit_learn(classes, folds):
    """The whole of voxelselector.py:41-53 for one voxel: StratifiedKFold splits, one-vs-one problems (libsvm's pair order,
    smaller label = +1), libsvm's vote -- mean accuracy equal to cross_val_score's, two to four conditions."""
    from sklearn import svm, model_selection
    rng = np.random.RandomState(10 * classes + folds)
    E = 36
    for shrinking in (False, True):
        for _ in range(6):
            K, lab = _svm_problem(rng, E, 120, 0.3, classes)
            lab = np.array([7, 2, 11, 5])[lab]                      # label values other than 0..k-1
            skf = model_selection.StratifiedKFold(n_splits=folds, shuffle=False)
            ref = model_selection.cross_val_score(svm.SVC(kernel="precomputed", shrinking=shrinking), K.astype(np.float64),
                                                  y=lab, cv=skf, n_jobs=1).mean()
            got, iters = orc.svm_cv(K, lab, folds, shrinking=shrinking)
            assert got == ref
            assert len(iters) == folds * classes * (classes - 1) // 2 and min(iters) >= 1
