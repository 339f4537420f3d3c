"""Epoch separation + the per-epoch normalisation (the "normalise prologue") on the GPU, and the host-side epoch
averaging of the activity-based (MVPA) path.

Mirrors the arithmetic of ``brainiak.fcma.preprocessing._separate_epochs`` (reference
preprocessing.py:41-92).  NIfTI loading / masking (preprocessing.py:156-232 via brainiak.image) is
out of scope: the functions here take the already masked ``[nVoxels, nTRs]`` activity arrays, or images that
yield their data through ``get_fdata()``, or plain arrays.

``generate_epochs_info``, ``prepare_mvpa_data`` and ``prepare_searchlight_mvpa_data`` (reference
preprocessing.py:235-414) average each epoch and z-score within subject.  They are not a hot path and run on the host
with the reference's numpy / scipy operations, so their output is bit-identical to the reference's.
"""
import logging
from enum import Enum

import numpy as np
from scipy.stats.mstats import zscore

from .. import _lib
from . import engine

__all__ = ["separate_epochs", "separate_epochs_device", "broadcast_epochs", "prepare_fcma_data", "RandomType",
           "generate_epochs_info", "prepare_mvpa_data", "prepare_searchlight_mvpa_data"]

logger = logging.getLogger(__name__)


def _epoch_slices(activity_data, epoch_list):
    """Enumerate (subject, condition, TR-mask) in the reference's order (preprocessing.py:71-77)."""
    out = []
    for sid in range(len(epoch_list)):
        epoch = epoch_list[sid]
        for cond in range(epoch.shape[0]):
            sub_epoch = epoch[cond, :, :]
            for eid in range(epoch.shape[1]):
                r = np.sum(sub_epoch[eid, :])
                if r > 0:
                    out.append((sid, cond, sub_epoch[eid, :] == 1))
    return out


def separate_epochs_device(activity_data, epoch_list, device=None):
    """Returns ``(epochs [E, Tmax, V] float32 CUDA (normalised, zero rows beyond T_e), T_e, labels)``."""
    import torch
    _lib.load()
    _lib.require_device()
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    slices = _epoch_slices(activity_data, epoch_list)
    raw, labels = [], []
    for sid, cond, m in slices:
        mat = np.ascontiguousarray(np.asarray(activity_data[sid], dtype=np.float32)[:, m].T)
        raw.append(mat)
        labels.append(cond)
    ep, T_e = engine.stack_epochs(raw, dev)
    engine.epoch_normalize_(ep, T_e)
    return ep, T_e, labels


def separate_epochs(activity_data, epoch_list, device=None):
    """Drop-in for ``_separate_epochs``: ``(raw_data: list of float32 [T_e, V], labels)``."""
    ep, T_e, labels = separate_epochs_device(activity_data, epoch_list, device)
    host = ep.cpu().numpy()
    return [np.ascontiguousarray(host[e, :T_e[e], :]) for e in range(len(T_e))], labels


_separate_epochs = separate_epochs


def broadcast_epochs(epochs, src=0):
    """NCCL broadcast of the normalised epoch tensor — the GPU replacement of the per-epoch
    ``comm.bcast`` loop of ``prepare_fcma_data`` (reference preprocessing.py:211-223).
    ``epochs`` must be allocated with the right shape on every rank."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(epochs, src=src)
    return epochs


class RandomType(Enum):
    """Randomisation of the voxel order within a subject (reference preprocessing.py:142-153)."""
    NORANDOM = 0
    REPRODUCIBLE = 1
    UNREPRODUCIBLE = 2


def _randomize_subject_list(data_list, random):
    """In-place voxel shuffles with the reference's seeding (preprocessing.py:95-139)."""
    if random == RandomType.REPRODUCIBLE:
        for i in range(len(data_list)):
            np.random.seed(i)
            np.random.shuffle(data_list[i])
    elif random == RandomType.UNREPRODUCIBLE:
        for data in data_list:
            np.random.shuffle(data)


def _mask_image(image, mask, data_type=np.float32):
    """brainiak.image.mask_image (reference image.py:107-140) for anything that yields a 3-D/4-D array: a nibabel
    SpatialImage (``get_fdata``) or a plain ``ndarray`` (NIfTI reading itself is out of scope here)."""
    data = image.get_fdata() if hasattr(image, "get_fdata") else np.asarray(image)
    mask = np.asarray(mask)
    if data.shape[:3] != mask.shape:
        raise ValueError("Image data and mask have different shapes.")
    return data.astype(data_type)[mask.astype(bool)]


def prepare_fcma_data(images, conditions, mask1, mask2=None, random=RandomType.NORANDOM, comm=None, device=None,
                      return_device=False):
    """Drop-in for ``brainiak.fcma.preprocessing.prepare_fcma_data`` (reference preprocessing.py:156-232): mask the
    images, separate and z-score the epochs, distribute them to all ranks.

    images: iterable of SpatialImage-likes (``get_fdata()``) or 4-D arrays, one per subject; conditions: list of
    ``[condition, nEpochs, nTRs]`` one-hot arrays; mask1 / mask2: boolean 3-D masks.  Rank 0 of ``torch.distributed``
    (the reference: rank 0 of ``comm``) does the masking; the per-epoch z-score (preprocessing.py:80-84) runs on its GPU
    (``fcma_epoch_normalize``), and instead of the per-epoch ``comm.bcast`` loop (preprocessing.py:211-223) the
    normalised ``[E, T, V]`` tensor goes to the other ranks with ONE NCCL broadcast over NVLink.  ``comm`` is accepted
    for signature compatibility and ignored (torch.distributed's default group is used).

    Returns ``(raw_data1, raw_data2, labels)`` like the reference: lists of float32 ``[epoch length, nVoxels]`` arrays
    (``raw_data2`` is None without ``mask2``).  ``return_device=True`` returns device tensors instead:
    ``((epochs1, T_e), (epochs2, T_e) | None, labels)`` with ``epochs`` = float32 CUDA ``[E, Tmax, V]``."""
    import torch
    import torch.distributed as dist
    _lib.load()
    _lib.require_device()
    multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    rank = dist.get_rank() if multi else 0
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    sets, labels, meta = [], [], None
    if rank == 0:
        masks = (mask1,) if mask2 is None else (mask1, mask2)
        per_mask = [[] for _ in masks]
        for image in images:
            for k, mk in enumerate(masks):
                per_mask[k].append(_mask_image(image, mk))
        # the reference shuffles mask 2's data first, then mask 1's (preprocessing.py:196-203)
        for k in reversed(range(len(masks))):
            _randomize_subject_list(per_mask[k], random)
        for k in range(len(masks)):
            ep, T_e, labels = separate_epochs_device(per_mask[k], conditions, dev)
            sets.append((ep, T_e))
        meta = [(tuple(ep.shape), T_e) for ep, T_e in sets] + [list(labels)]
    if multi:
        box = [meta]
        dist.broadcast_object_list(box, src=0)
        meta = box[0]
        labels = meta[-1]
        for k, (shape, T_e) in enumerate(meta[:-1]):
            if rank != 0:
                sets.append((torch.empty(shape, dtype=torch.float32, device=dev), T_e))
            dist.broadcast(sets[k][0], src=0)
    if return_device:
        return sets[0], (sets[1] if len(sets) > 1 else None), labels
    out = []
    for ep, T_e in sets:
        host = ep.cpu().numpy()
        out.append([np.ascontiguousarray(host[e, :T_e[e], :]) for e in range(len(T_e))])
    return out[0], (out[1] if len(out) > 1 else None), labels


# ------------------------------------------------------------------ activity-based (MVPA) preprocessing, on the host
def generate_epochs_info(epoch_list):
    """Epochs of ``epoch_list`` (one ``[condition, nEpochs, nTRs]`` 0/1 array per subject, every epoch a contiguous run
    of TRs) as a list of ``(label, sid, start, end)``, ``end`` exclusive, in the reference's order: subject, then
    condition, then epoch (preprocessing.py:235-271)."""
    epoch_info = []
    for sid, epoch in enumerate(epoch_list):
        for cond in range(epoch.shape[0]):
            sub_epoch = epoch[cond, :, :]
            for eid in range(epoch.shape[1]):
                r = np.sum(sub_epoch[eid, :])
                if r > 0:
                    start = np.nonzero(sub_epoch[eid, :])[0][0]
                    epoch_info.append((cond, sid, start, start + r))
    return epoch_info


def _zscore_subjects_(processed_data, subject_count):
    """z-score the epochs of each subject along the last axis, in place (subjects with one epoch are left as they are),
    then ``nan_to_num`` (a constant voxel has sigma 0)."""
    axis = processed_data.ndim - 1
    cur_epoch = 0
    for i in subject_count:
        if i > 1:
            processed_data[..., cur_epoch:cur_epoch + i] = \
                zscore(processed_data[..., cur_epoch:cur_epoch + i], axis=axis, ddof=0)
        cur_epoch += i
    return np.nan_to_num(processed_data)


def prepare_mvpa_data(images, conditions, mask):
    """Drop-in for ``brainiak.fcma.preprocessing.prepare_mvpa_data`` (reference preprocessing.py:274-325): mask each
    subject's image, average the activity within every epoch and z-score the epochs within subject.

    Returns ``(processed_data, labels)``: float64 ``[num_voxels, num_epochs]`` and float64 ``[num_epochs]``."""
    activity_data = [_mask_image(image, mask, np.float32) for image in images]
    epoch_info = generate_epochs_info(conditions)
    num_epochs = len(epoch_info)
    (d1, _) = activity_data[0].shape
    processed_data = np.empty([d1, num_epochs])
    labels = np.empty(num_epochs)
    subject_count = [0]
    cur_sid = -1
    for idx, epoch in enumerate(epoch_info):
        labels[idx] = epoch[0]
        if cur_sid != epoch[1]:
            subject_count.append(0)
            cur_sid = epoch[1]
        subject_count[-1] += 1
        processed_data[:, idx] = np.mean(activity_data[cur_sid][:, epoch[2]:epoch[3]], axis=1)
    return _zscore_subjects_(processed_data, subject_count), labels


def prepare_searchlight_mvpa_data(images, conditions, data_type=np.float32, random=RandomType.NORANDOM):
    """Drop-in for ``brainiak.fcma.preprocessing.prepare_searchlight_mvpa_data`` (reference preprocessing.py:328-414):
    the input of ``MVPAVoxelSelector``.  Averages the activity within every epoch and z-scores the epochs within
    subject, keeping the 3-D brain; subjects are processed one at a time.  ``random`` shuffles each subject's voxels
    (REPRODUCIBLE: seeded with the subject index).

    Returns ``(processed_data, labels)``: ``data_type`` ``[X, Y, Z, num_epochs]`` and float64 ``[num_epochs]``."""
    epoch_info = generate_epochs_info(conditions)
    num_epochs = len(epoch_info)
    processed_data = None
    logger.info('there are %d subjects, and in total %d epochs', len(conditions), num_epochs)
    labels = np.empty(num_epochs)
    for idx, epoch in enumerate(epoch_info):
        labels[idx] = epoch[0]
    subject_count = np.zeros(len(conditions), dtype=np.int32)
    for sid, f in enumerate(images):
        data = (f.get_fdata() if hasattr(f, "get_fdata") else np.asarray(f)).astype(data_type)
        if data.ndim != 4:
            raise ValueError("image %d is not 4-D" % sid)
        [d1, d2, d3, d4] = data.shape
        if random != RandomType.NORANDOM:
            data = data.reshape((d1 * d2 * d3, d4))
            if random == RandomType.REPRODUCIBLE:
                np.random.seed(sid)
            np.random.shuffle(data)
            data = data.reshape((d1, d2, d3, d4))
        if processed_data is None:
            processed_data = np.empty([d1, d2, d3, num_epochs], dtype=data_type)
        for idx, epoch in enumerate(epoch_info):
            if sid == epoch[1]:
                subject_count[sid] += 1
                processed_data[:, :, :, idx] = np.mean(data[:, :, :, epoch[2]:epoch[3]], axis=3)
    return _zscore_subjects_(processed_data, subject_count), labels
