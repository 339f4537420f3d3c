#!/usr/bin/env python
"""Generate tests/golden/clf_w*.npz, the Classifier fixtures at multi-tile shapes, by running the UNMODIFIED reference
Classifier (oracle/_ref, built by oracle/build_ref.sh) on the CPU.

The inputs are seeded dyadic epochs (brainiak_b200.fcma.synthetic.make_dyadic_epochs: every correlation exact in fp32,
so r is the same in any summation order); the tests regenerate them from the seeds (``clf_inputs``) and each file
stores a probe of them and the reference's outputs: the shrunk kernel of the fitted samples, ``num_digits_``,
``test_data_``, ``decision_function``, ``predict`` and ``score``.

* w1: one mask of 640 voxels, E = 32, eps 8, portion mode (``num_processed_voxels = 200``), 24 training samples: the
  fit-time test samples are exactly one subject.
* w2: two masks of 300 and 700 voxels passed smaller-first, 40 samples, eps 5: a small-mask fit on the first 30, then
  ``predict`` / ``decision_function`` / ``score`` on the last 10.
* w3: two masks of 120 and 90 voxels, E = 100, eps 12 (4 trailing epochs), portion mode with 84 training samples.
* w4: ``LogisticRegression`` on two masks of 40 and 30 voxels, 24 samples, eps 4: fit on the first 16, predict the
  last 8.

Run from the repo root where the reference tree exists:

    bash oracle/build_ref.sh && python tests/golden/make_golden_clf_wide.py
"""
import os
import sys

import numpy as np
from sklearn import svm
from sklearn.linear_model import LogisticRegression

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, input_probe, reference, synthetic  # noqa: E402


def svc():
    return svm.SVC(kernel="precomputed", shrinking=False, C=1)


def clf_inputs(name):
    """(X, labels, eps, num_processed_voxels, split) of fixture ``name``, regenerated from the seeds.  X is the list of
    (data1, data2) pairs in the order given to the Classifier; ``split`` is num_training_samples (portion mode) or the
    number of samples fitted before predicting the rest."""
    if name == "w1":
        raw, labels = synthetic.make_dyadic_epochs(640, 20, 32, seed=8080, informative=60)
        return list(zip(raw, raw)), labels, 8, 200, 24
    if name == "w2":
        big, labels = synthetic.make_dyadic_epochs(700, 16, 40, seed=8181, informative=80)
        small, _ = synthetic.make_dyadic_epochs(300, 16, 40, seed=8282, informative=40)
        return list(zip(small, big)), labels, 5, 2000, 30
    if name == "w3":
        a, labels = synthetic.make_dyadic_epochs(120, 24, 100, seed=8383, informative=20)
        b, _ = synthetic.make_dyadic_epochs(90, 24, 100, seed=8484, informative=15)
        return list(zip(a, b)), labels, 12, 50, 84
    if name == "w4":
        a, labels = synthetic.make_dyadic_epochs(40, 12, 24, seed=8585, informative=8)
        b, _ = synthetic.make_dyadic_epochs(30, 12, 24, seed=8686, informative=6)
        return list(zip(a, b)), labels, 4, 2000, 16
    raise ValueError(name)


def fit_kernel(m, X, eps):
    """The reference's shrunk kernel of the samples X and its digit count (classifier.py:279-348 in one portion)."""
    X1, X2 = zip(*X)
    if X1[0].shape[1] < X2[0].shape[1]:
        X1, X2 = X2, X1
    c = m.Classifier(svc(), epochs_per_subj=eps)
    c.num_voxels_, c.num_features_, c.num_samples_ = X1[0].shape[1], X1[0].shape[1] * X2[0].shape[1], len(X1)
    K, _ = c._compute_kernel_matrix_in_portion(list(X1), list(X2))
    return K, c.num_digits_


def save(name):
    m = reference.load()
    X, labels, eps, npv, split = clf_inputs(name)
    out = dict(probe=input_probe([x for x, _ in X]), probe2=input_probe([y for _, y in X]), labels=np.array(labels),
               eps=eps)
    if name == "w4":
        c = m.Classifier(LogisticRegression(), epochs_per_subj=eps)
        c.fit(X[:split], labels[:split])
        test = X[split:]
        out.update(decision=c.decision_function(test), predict=c.predict(test), score=c.score(test, labels[split:]))
    elif name == "w2":
        c = m.Classifier(svc(), num_processed_voxels=npv, epochs_per_subj=eps)
        c.fit(X[:split], labels[:split])
        out["kernel"], _ = fit_kernel(m, X[:split], eps)
        test = X[split:]
        out.update(num_digits=c.num_digits_, decision=c.decision_function(test), predict=c.predict(test),
                   test_data=c.test_data_.copy(), score=c.score(test, labels[split:]))
    else:
        c = m.Classifier(svc(), num_processed_voxels=npv, epochs_per_subj=eps)
        c.fit(X, labels, num_training_samples=split)
        out["kernel"], nd = fit_kernel(m, X, eps)
        assert nd == c.num_digits_
        out.update(num_digits=c.num_digits_, test_data=c.test_data_.copy(), decision=c.decision_function(),
                   predict=c.predict(), score=c.score(None, labels[split:]))
    np.savez_compressed(os.path.join(OUT, "clf_%s.npz" % name), **out)
    print(name, "predict", out["predict"], "score", out["score"], "digits", out.get("num_digits"))


if __name__ == "__main__":
    for name in sys.argv[1:] or ["w1", "w2", "w3", "w4"]:
        save(name)
