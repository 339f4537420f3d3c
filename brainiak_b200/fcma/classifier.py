"""Full Correlation Matrix Analysis (FCMA) — correlation-based classification on H100.

Drop-in for ``brainiak.fcma.classifier.Classifier`` (reference classifier.py:37-690): an sklearn
``BaseEstimator`` with the same constructor arguments, fitted attributes and
``fit / predict / decision_function / score`` behaviour.  The native stages run on the GPU through
libfcma_b200.so:

* ``_prepare_corerelation_data``  (classifier.py:125-182, a9)  -> wgmma correlation GEMM
* ``_normalize_correlation_data`` (classifier.py:184-220, a10) -> Fisher-z + z-score kernel
* ``_compute_kernel_matrix_in_portion`` (classifier.py:279-348, a11) -> fused GEMM -> normalise ->
  ``K += Z Z^T`` without ever materialising the ``[E, rows, V2]`` correlation block on the host
* ``_prepare_test_data``          (classifier.py:222-277, a12) -> NT GEMM against the training features

Large masks (SURVEY §8f rank 4): after a portion-mode fit the reference cannot ``predict(X)`` new data because it would
need ``training_data_`` = ``[n_train, V1*V2]`` features (320 GB at V = 50 000).  Here the classifier keeps references to
the raw TRAINING epochs instead (1.3 GB) and ``predict`` / ``decision_function`` stream the test-vs-train similarity
portion by portion on the GPU (``_streamed_similarity``) without ever materialising the features.
"""
import logging
import time

import numpy as np
import sklearn
import sklearn.svm
from sklearn.base import BaseEstimator

from .. import _lib
from . import engine

logger = logging.getLogger(__name__)

__all__ = ["Classifier"]


def _is_precomputed_svc(clf):
    return isinstance(clf, sklearn.svm.SVC) and clf.kernel == 'precomputed'


# the kernel matrix of more than 64 samples is formed by k_syrk_simt, which holds 64 (E + 1) floats of shared memory
# per block, at most 200 KB
MAX_KERNEL_SAMPLES = 799


def _check_kernel_samples(E, what):
    if E > MAX_KERNEL_SAMPLES:
        raise ValueError("%s: %d samples, but the kernel matrix of SVC(kernel='precomputed') is limited to %d samples"
                         % (what, E, MAX_KERNEL_SAMPLES))


class Classifier(BaseEstimator):
    """Correlation-based classification component of FCMA (H100 engine).

    Parameters
    ----------
    clf, num_processed_voxels=2000, epochs_per_subj=0:
        as in the reference (classifier.py:115-123).
    precision: str, default 'fp32'
        operand precision of the correlation contraction ('fp32' = fp32-faithful 3-product split,
        see VoxelSelector).
    device: optional CUDA device

    With ``SVC(kernel='precomputed')`` the kernel matrix holds at most ``MAX_KERNEL_SAMPLES`` = 799 samples: the
    samples of ``fit``, and after a fit in portions (``num_processed_voxels`` below the larger mask) the training samples
    of fit's subjects plus the samples given to ``predict`` / ``decision_function``.  More raise ``ValueError``.

    Attributes (classifier.py:68-114)
    ----------
    training_data_, test_raw_data_, test_data_, num_voxels_, num_features_, num_samples_, num_digits_
    """

    def __init__(self, clf, num_processed_voxels=2000, epochs_per_subj=0, precision="fp32",
                 device=None):
        self.clf = clf
        self.num_processed_voxels = num_processed_voxels
        self.epochs_per_subj = epochs_per_subj
        self.precision = precision
        self.device = device
        self.num_digits_ = 0
        self._train_raw_ = None
        return

    # ------------------------------------------------------------------ device helpers
    def _torch_device(self):
        import torch
        if self.device is not None:
            return torch.device(self.device)
        return torch.device("cuda", torch.cuda.current_device())

    def _pack_pair(self, X1, X2):
        _lib.load()
        _lib.require_device()
        dev = self._torch_device()
        ep1, T1 = engine.stack_epochs(list(X1), dev)
        prec = engine.resolve_precision(self.precision, ep1)
        same = len(X1) == len(X2) and all(a is b for a, b in zip(X1, X2))
        if same:
            op1 = engine.pack_epochs(ep1, T1, prec)
            return op1, op1
        ep2, T2 = engine.stack_epochs(list(X2), dev)
        if T1 != T2:
            raise AssertionError('the numbers of TRs of X1 and X2 are not identical')
        if engine.resolve_precision(self.precision, ep2) != prec:
            prec = "tf32x3"
        return engine.pack_epochs(ep1, T1, prec), engine.pack_epochs(ep2, T2, prec)

    # ------------------------------------------------------------------ reference stage methods
    def _prepare_corerelation_data(self, X1, X2, start_voxel=0, num_processed_voxels=None):
        """a9: correlation between ``num_processed_voxels`` voxels of X1 and all voxels of X2.

        Returns float32 numpy ``[len(X), num_processed_voxels, num_voxels2]`` (classifier.py:125-182)."""
        num_samples = len(X1)
        assert num_samples > 0, 'at least one sample is needed for correlation computation'
        num_voxels1 = X1[0].shape[1]
        num_voxels2 = X2[0].shape[1]
        assert num_voxels1 * num_voxels2 == self.num_features_, \
            'the number of features provided by the input data ' \
            'does not match the number of features defined in the model'
        assert X1[0].shape[0] == X2[0].shape[0], \
            'the numbers of TRs of X1 and X2 are not identical'
        if num_processed_voxels is None:
            num_processed_voxels = num_voxels1
        op1, op2 = self._pack_pair(X1, X2)
        corr = engine.corr_block(op1, op2, start_voxel, num_processed_voxels, layout=1)
        logger.debug('correlation computation done')
        return corr.cpu().numpy()

    def _normalize_correlation_data(self, corr_data, norm_unit):
        """a10: Fisher-transform and z-score every ``norm_unit`` samples if ``norm_unit > 1``
        (classifier.py:184-220)."""
        import torch
        if norm_unit > 1:
            num_samples = len(corr_data)
            [_, d2, d3] = corr_data.shape
            c = np.ascontiguousarray(corr_data, dtype=np.float32).reshape(1, num_samples, d2 * d3)
            t = torch.from_numpy(c).to(self._torch_device())
            engine.within_subject_norm_(t, norm_unit)
            normalized_corr_data = t.cpu().numpy().reshape(num_samples, d2, d3)
            logger.debug('normalization done')
        else:
            normalized_corr_data = corr_data
        return normalized_corr_data

    def _prepare_test_data(self, corr_data):
        """a12: similarity vectors of the test samples against the training features, or the
        reshaped features for non-kernel classifiers (classifier.py:222-277)."""
        import torch
        num_test_samples = corr_data.shape[0]
        assert num_test_samples > 0, 'at least one test sample is needed'
        if _is_precomputed_svc(self.clf):
            assert self.training_data_ is not None, \
                'when using precomputed kernel of SVM, all training data must be provided'
            dev = self._torch_device()
            test = torch.from_numpy(np.ascontiguousarray(
                corr_data.reshape(num_test_samples, self.num_features_), dtype=np.float32)).to(dev)
            train = torch.from_numpy(np.ascontiguousarray(self.training_data_, dtype=np.float32)).to(dev)
            data = engine.gemm_nt(test, train).cpu().numpy()
            num_digits = self.num_digits_
            if num_digits > 2:
                proportion = 10 ** (2 - num_digits)
                data *= proportion
            logger.debug('similarity vectors computation done')
        else:
            data = corr_data.reshape(num_test_samples, self.num_features_)
        return data

    def _compute_kernel_matrix_in_portion(self, X1, X2):
        """a11: kernel matrix for SVC(kernel='precomputed'), portion by portion
        (classifier.py:279-348).  Returns ``(kernel_matrix [E, E], normalized_corr_data)``;
        the second item is the ``[1, E, rows*V2]`` features of the LAST portion, kept only when a
        single portion covers all voxels (it becomes ``training_data_``)."""
        import torch
        E = self.num_samples_
        _check_kernel_samples(E, "fit")
        op1, op2 = self._pack_pair(X1, X2)
        num_voxels2 = X2[0].shape[1]
        single = self.num_processed_voxels >= self.num_voxels_
        normalized_corr_data = None
        if single:
            # small-mask use: the features are needed later for prediction -> materialise them
            corr = engine.corr_block(op1, op2, 0, self.num_voxels_, layout=1).contiguous()
            flat = corr.view(1, E, self.num_voxels_ * num_voxels2)
            if self.epochs_per_subj > 1:
                engine.within_subject_norm_(flat, self.epochs_per_subj)
            K = engine.kernel_matrices(flat, sum_over_rows=True)
            normalized_corr_data = flat.cpu().numpy()
        else:
            # portion mode: the reference accumulates portion by portion to bound host memory; on
            # the GPU the block size is bounded by the scratch buffer and nothing is materialised
            K = torch.zeros((E, E), dtype=torch.float32, device=op1.device)
            engine.classifier_kernel(op1, op2, 0, self.num_voxels_, self.epochs_per_subj, out=K)
        kernel_matrix = K.cpu().numpy()
        num_digits = len(str(int(kernel_matrix[0, 0])))
        self.num_digits_ = num_digits
        if num_digits > 2:
            proportion = 10 ** (2 - num_digits)
            kernel_matrix *= proportion
        return kernel_matrix, normalized_corr_data

    def _generate_training_data(self, X1, X2, num_training_samples):
        """classifier.py:350-424."""
        if not _is_precomputed_svc(self.clf):
            corr_data = self._prepare_corerelation_data(X1, X2)
            normalized_corr_data = self._normalize_correlation_data(corr_data, self.epochs_per_subj)
            data = normalized_corr_data.reshape(self.num_samples_, self.num_features_)
            self.training_data_ = None
        else:  # SVM with precomputed kernel
            if self.num_processed_voxels < self.num_voxels_:
                if num_training_samples is None:
                    raise RuntimeError('the kernel matrix will be '
                                       'computed portion by portion, '
                                       'the test samples must be predefined '
                                       'by specifying '
                                       'num_training_samples')
                if num_training_samples >= self.num_samples_:
                    raise ValueError('the number of training samples '
                                     'must be smaller than '
                                     'the number of total samples')
            data, normalized_corr_data = self._compute_kernel_matrix_in_portion(X1, X2)
            if self.num_processed_voxels >= self.num_voxels_:
                self.training_data_ = normalized_corr_data.reshape(self.num_samples_,
                                                                   self.num_features_)
                self._train_raw_ = None
            else:
                self.training_data_ = None
                # references (no copies) to the raw training epochs: what streamed prediction needs instead of the
                # [n_train, V1*V2] features.  fit normalised the training samples within subjects of epochs_per_subj
                # over all fit samples, so a subject cut by n_train is kept whole: its first samples' features depend
                # on the fit-time test samples that share the subject
                n_train = num_training_samples if num_training_samples is not None else self.num_samples_
                eps = self.epochs_per_subj
                n_span = n_train if eps <= 1 else min(self.num_samples_, -(-n_train // eps) * eps)
                self._train_raw_ = (list(X1[:n_span]), list(X2[:n_span]))
                self._num_train_ = n_train
            logger.debug('kernel computation done')
        return data

    # ------------------------------------------------------------------ estimator API
    def fit(self, X, y, num_training_samples=None):
        """Use correlation data to train a model (classifier.py:426-504)."""
        time1 = time.time()
        assert len(X) == len(y), 'the number of samples must be equal to the number of labels'
        for x in X:
            assert len(x) == 2, 'there must be two parts for each correlation computation'
        X1, X2 = zip(*X)
        if not _is_precomputed_svc(self.clf):
            if num_training_samples is not None:
                num_training_samples = None
                logger.warning('num_training_samples should not be set for classifiers '
                               'other than SVM with precomputed kernels')
        num_samples = len(X1)
        num_voxels1 = X1[0].shape[1]
        num_voxels2 = X2[0].shape[1]
        if num_voxels1 < num_voxels2:
            X1, X2 = X2, X1
            num_voxels1, num_voxels2 = num_voxels2, num_voxels1
        self.num_voxels_ = num_voxels1
        self.num_features_ = num_voxels1 * num_voxels2
        self.num_samples_ = num_samples

        data = self._generate_training_data(X1, X2, num_training_samples)

        if num_training_samples is not None:
            self.test_raw_data_ = None
            self.test_data_ = data[num_training_samples:, 0:num_training_samples]
            data = data[0:num_training_samples, 0:num_training_samples]
        self.clf = self.clf.fit(data, y[0:num_training_samples])
        if num_training_samples is None:
            self.test_raw_data_ = None
            self.test_data_ = None
        logger.info('training done, takes %.2f s', time.time() - time1)
        return self

    def _features_for_prediction(self, X):
        for x in X:
            assert len(x) == 2, 'there must be two parts for each correlation computation'
        X1, X2 = zip(*X)
        num_voxels1 = X1[0].shape[1]
        num_voxels2 = X2[0].shape[1]
        assert len(X1) == len(X2), 'the list lengths do not match'
        if num_voxels1 < num_voxels2:
            X1, X2 = X2, X1
            num_voxels1, num_voxels2 = num_voxels2, num_voxels1
        assert self.num_features_ == num_voxels1 * num_voxels2, \
            'the number of features does not match the model'
        num_test_samples = len(X1)
        self.test_raw_data_ = X
        if _is_precomputed_svc(self.clf) and self.training_data_ is None and \
                getattr(self, "_train_raw_", None) is not None:
            self.test_data_ = self._streamed_similarity(X1, X2)
            return
        corr_data = self._prepare_corerelation_data(X1, X2)
        normalized_corr_data = self._normalize_correlation_data(corr_data, num_test_samples)
        self.test_data_ = self._prepare_test_data(normalized_corr_data)

    def _streamed_similarity(self, X1, X2, max_bytes=8 << 30):
        """Test-vs-train similarity ``[n_test, n_train]`` for large masks, never materialising the features
        (the reference's ``_prepare_test_data``, classifier.py:222-277, needs ``training_data_``).

        The training and the test epochs form one sample list; per portion of voxel rows the tensor-core GEMM writes
        the correlation block ``[samples, rows, V2]`` (a9), the training part is normalised within subject with
        ``epochs_per_subj`` as ``fit`` does (classifier.py:325-327), the test part over all test samples as ``predict``
        does (classifier.py:554-556), and ``K += Z Z^T`` accumulates the Gram matrix over the portions (a11); its
        test x train block, scaled with the ``num_digits_`` of the training kernel, is the similarity.  The training
        part is the fit samples up to the end of the subject of the last training sample (``_train_raw_``), so every
        training sample is z-scored with the same epochs as in ``fit``; only the first ``n_train`` columns are used."""
        import torch
        tr1, tr2 = self._train_raw_
        n_span, n_test = len(tr1), len(X1)
        n_train = getattr(self, "_num_train_", n_span)
        if tr1[0].shape[1] != X1[0].shape[1]:        # fit() may have swapped the masks so that X1 is the larger one
            tr1, tr2 = tr2, tr1
        Es = n_span + n_test
        _check_kernel_samples(Es, "the training samples of fit's subjects and the test samples")
        op1, op2 = self._pack_pair(list(tr1) + list(X1), list(tr2) + list(X2))
        V1, V2 = op1.V, op2.V
        rows = int(max(1, min(self.num_processed_voxels, V1, max_bytes // (Es * V2 * 4))))
        K = torch.zeros((Es, Es), dtype=torch.float32, device=op1.device)
        for start in range(0, V1, rows):
            nb = min(rows, V1 - start)
            corr = engine.corr_block(op1, op2, start, nb, layout=1)                    # [Es, nb, V2]
            if self.epochs_per_subj > 1:
                engine.within_subject_norm_(corr[:n_span].view(1, n_span, nb * V2), self.epochs_per_subj)
            if n_test > 1:
                engine.within_subject_norm_(corr[n_span:].view(1, n_test, nb * V2), n_test)
            engine.kernel_matrices(corr.view(1, Es, nb * V2), beta=1.0, out=K, sum_over_rows=True)
        data = K[n_span:, :n_train].cpu().numpy()
        if self.num_digits_ > 2:
            data *= 10 ** (2 - self.num_digits_)
        logger.debug('streamed similarity vectors computation done')
        return np.ascontiguousarray(data)

    def predict(self, X=None):
        """Use a trained model to predict correlation data (classifier.py:506-566)."""
        time1 = time.time()
        if X is not None:
            self._features_for_prediction(X)
        y_pred = self.clf.predict(self.test_data_)
        logger.info('prediction done, takes %.2f s', time.time() - time1)
        return y_pred

    def _is_equal_to_test_raw_data(self, X):
        """classifier.py:568-595."""
        if self.test_raw_data_ is None or len(X) != len(self.test_raw_data_):
            return False
        X1, X2 = zip(*X)
        c1, c2 = zip(*self.test_raw_data_)
        for new, old in zip(X1, c1):
            if not np.array_equal(new, old):
                return False
        for new, old in zip(X2, c2):
            if not np.array_equal(new, old):
                return False
        return True

    def decision_function(self, X=None):
        """Decision values of the prediction (classifier.py:597-650)."""
        if X is not None and not self._is_equal_to_test_raw_data(X):
            self._features_for_prediction(X)
        confidence = self.clf.decision_function(self.test_data_)
        return confidence

    def score(self, X, y, sample_weight=None):
        """Mean accuracy on the given test data and labels (classifier.py:652-690)."""
        from sklearn.metrics import accuracy_score
        if _is_precomputed_svc(self.clf) and self.training_data_ is None:
            result = accuracy_score(y, self.predict(), sample_weight=sample_weight)
        else:
            result = accuracy_score(y, self.predict(X), sample_weight=sample_weight)
        return result
