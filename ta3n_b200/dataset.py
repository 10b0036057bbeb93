"""Feature input pipeline for the path (SURVEY 8f row n3): what sits in front of `VideoModel.forward`.

The reference (`dataset.py`) keeps one `.t7` file per frame and `torch.load`s num_segments of them per clip,
per iteration -- on real data its training loop is bound by those file opens (5 per clip), not by the model.
This module offers

* `TSNDataSet` / `VideoRecord`: drop-in for `dataset.py:16-152` (same constructor, same index rules, same
  `(num_segments*new_length, feat_dim) tensor, label` items), for code that keeps the per-frame files;
* `pack_list()` + `PackedTSNDataSet`: because `main.py:171-196` builds every split -- training included -- with
  `random_shift=False, test_mode=True`, the frames a clip contributes are a pure function of its length.  They
  are gathered ONCE into a `(num_videos, T, feat_dim)` fp32 `.npy` shard that is memory-mapped afterwards;
* `PairedFeatureLoader`: the `enumerate(zip(source_loader, target_loader))` of `main.py:343-346` with
  `RandomSampler` order, assembling every paired mini-batch directly into (pinned) staging buffers on a
  background thread, ready for `TrainStep.prefetch()`;
* `DeviceFeatureBank` + `DevicePairedSampler`: the same epochs with the shards resident in device memory; each
  mini-batch is gathered by the first launch of the captured step (`TrainStep(..., sampler=...)`);
* `DeviceEvalSampler`: the validation loader (one bank, dataset order) for `evaluate.EvalStep(..., sampler=...)`.

Both paired paths draw their epochs from `paired_epoch_plan`, so that one seed gives the same batches on either.
"""
from __future__ import annotations

import json
import os
import queue
import threading
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.utils.data as data

_RGB_LIKE = ("RGB", "RGBDiff", "RGBDiff2", "RGBDiffplus")


# ---- which frames of a video are used ----------------------------------------------------------------
def _centre_ticks(num_select: int, num_segments: int) -> np.ndarray:
    # centre of each of num_segments equal spans of [0, num_select): floor(tick/2 + tick*x), same float ops
    # and order as dataset.py:98-99 / :109-110
    tick = float(num_select) / float(num_segments)
    return np.floor(tick / 2.0 + tick * np.arange(num_segments, dtype=np.float64)).astype(np.int64)


def test_segment_indices(num_frames: int, num_segments: int, new_length: int = 1) -> np.ndarray:
    """1-based start frames, `_get_test_indices` (dataset.py:103-116).  A clip shorter than
    num_segments + new_length - 1 uses its selectable frames in order and repeats the last one."""
    num_select = num_frames - new_length + 1
    if num_frames >= num_segments + new_length - 1:
        return _centre_ticks(num_select, num_segments) + 1
    if num_select <= 0:
        raise IndexError(f"video with {num_frames} frames is shorter than new_length={new_length}")   # as the reference
    return np.minimum(np.arange(num_segments, dtype=np.int64), num_select - 1) + 1


def val_segment_indices(num_frames: int, num_segments: int, new_length: int = 1) -> np.ndarray:
    """`_get_val_indices` (dataset.py:92-101): as the test rule, but a too-short clip uses frame 1 throughout."""
    if num_frames >= num_segments + new_length - 1:
        return _centre_ticks(num_frames - new_length + 1, num_segments) + 1
    return np.ones(num_segments, dtype=np.int64)


def random_segment_indices(num_frames: int, num_segments: int, new_length: int = 1) -> np.ndarray:
    """`_sample_indices` (dataset.py:77-90): one random frame per segment.  Draws from numpy's global RandomState
    with the reference's calls in the reference's order, so `numpy.random.seed` reproduces its sequences."""
    span = (num_frames - new_length + 1) // num_segments
    if span > 0:
        return np.arange(num_segments, dtype=np.int64) * span + np.random.randint(span, size=num_segments) + 1
    if num_frames > num_segments:
        return np.sort(np.random.randint(num_frames - new_length + 1, size=num_segments)).astype(np.int64) + 1
    return np.ones(num_segments, dtype=np.int64)


def expand_frames(starts: Sequence[int], num_frames: int, new_length: int = 1) -> List[int]:
    """`get` (dataset.py:128-140): new_length consecutive frames per start, not running past the last frame."""
    frames = []
    for s in starts:
        p = int(s)
        for _ in range(new_length):
            frames.append(p)
            p += 1 if p < num_frames else 0
    return frames


class VideoRecord(object):
    """One line `path num_frames label` of a list file (dataset.py:16-30)."""

    def __init__(self, row):
        self._data = row

    @property
    def path(self):
        return self._data[0]

    @property
    def num_frames(self):
        return int(self._data[1])

    @property
    def label(self):
        return int(self._data[2])


def _read_list(list_file: str, num_dataload: Optional[int]) -> List[VideoRecord]:
    with open(list_file) as f:
        records = [VideoRecord(line.strip().split(" ")) for line in f if line.strip()]
    if not records:
        raise ValueError(f"{list_file}: empty list")
    if num_dataload is None:
        return records
    # dataset.py:70-75: tile the list to exactly num_dataload items (the shorter domain is repeated, main.py:145-153)
    reps, left = divmod(int(num_dataload), len(records))
    return records * reps + records[:left]


class TSNDataSet(data.Dataset):
    """Drop-in for the reference's `TSNDataSet` (dataset.py:33-152): per-frame `.t7` feature files."""

    def __init__(self, root_path, list_file, num_dataload, num_segments=3, new_length=1, modality='RGB',
                 image_tmpl='img_{:05d}.t7', transform=None, force_grayscale=False, random_shift=True,
                 test_mode=False):
        self.root_path = root_path
        self.list_file = list_file
        self.num_segments = num_segments
        self.new_length = new_length + (1 if modality in ('RGBDiff', 'RGBDiff2', 'RGBDiffplus') else 0)   # :48-49
        self.modality = modality
        self.image_tmpl = image_tmpl
        self.transform = transform
        self.random_shift = random_shift
        self.test_mode = test_mode
        self.num_dataload = num_dataload
        self.video_list = _read_list(list_file, num_dataload)

    def segment_indices(self, record: VideoRecord) -> np.ndarray:
        if self.test_mode:
            return test_segment_indices(record.num_frames, self.num_segments, self.new_length)
        rule = random_segment_indices if self.random_shift else val_segment_indices
        return rule(record.num_frames, self.num_segments, self.new_length)

    def _load_feature(self, directory, idx):
        if self.modality in _RGB_LIKE:
            return [torch.load(os.path.join(directory, self.image_tmpl.format(idx)))]
        if self.modality == 'Flow':
            return [torch.load(os.path.join(directory, self.image_tmpl.format(axis, idx))) for axis in ('x', 'y')]
        raise ValueError(f"unknown modality {self.modality}")

    def get(self, record, indices):
        feats = []
        for p in expand_frames(indices, record.num_frames, self.new_length):
            feats.extend(self._load_feature(record.path, p))
        return torch.stack(feats), record.label

    def __getitem__(self, index):
        record = self.video_list[index]
        return self.get(record, self.segment_indices(record))

    def __len__(self):
        return len(self.video_list)


# ---- packed shards -----------------------------------------------------------------------------------
def pack_list(list_file: str, out_path: str, num_segments: int, new_length: int = 1, modality: str = 'RGB',
              image_tmpl: str = 'img_{:05d}.t7', rule: str = 'test') -> Tuple[int, int, int]:
    """Gather the frames every clip of `list_file` contributes under the deterministic index rule into one
    `(num_videos, num_segments*new_length, feat_dim)` float32 `.npy` file (+ `<out_path>.json` with labels,
    paths and the rule).  `rule`: 'test' (what main.py uses for all splits) or 'val'.  Returns the shape."""
    if rule not in ('test', 'val'):
        raise ValueError("only the deterministic rules can be packed ('test' or 'val')")
    src = TSNDataSet("", list_file, num_dataload=None, num_segments=num_segments, new_length=new_length,
                     modality=modality, image_tmpl=image_tmpl, random_shift=False, test_mode=(rule == 'test'))
    first, _ = src[0]
    shape = (len(src),) + tuple(first.shape)
    out = np.lib.format.open_memmap(out_path, mode='w+', dtype=np.float32, shape=shape)
    labels, paths, lengths = [], [], []
    for i in range(len(src)):
        x, y = (first, src.video_list[0].label) if i == 0 else src[i]
        if tuple(x.shape) != shape[1:]:
            raise ValueError(f"{src.video_list[i].path}: feature shape {tuple(x.shape)} != {shape[1:]}")
        out[i] = x.to(torch.float32).numpy()
        labels.append(int(y))
        paths.append(src.video_list[i].path)
        lengths.append(src.video_list[i].num_frames)
    out.flush()
    del out
    with open(out_path + ".json", "w") as f:
        json.dump({"list_file": os.path.abspath(list_file), "num_segments": num_segments, "new_length": src.new_length,
                   "modality": modality, "rule": rule, "labels": labels, "paths": paths, "num_frames": lengths}, f)
    return shape


class PackedTSNDataSet(data.Dataset):
    """The same items as `TSNDataSet(..., random_shift=False, test_mode=True)` served from a packed shard:
    one memory-mapped row copy instead of num_segments `torch.load` calls."""

    def __init__(self, packed_path: str, num_dataload: Optional[int] = None):
        self.features = np.load(packed_path, mmap_mode='r')
        with open(packed_path + ".json") as f:
            self.meta = json.load(f)
        if len(self.meta["labels"]) != self.features.shape[0]:
            raise ValueError("shard and metadata disagree on the number of videos")
        if self.features.dtype != np.float32 or self.features.ndim != 3:
            raise ValueError(f"{packed_path}: expected a (videos, frames, feat_dim) float32 shard as written by pack_list, "
                             f"got {self.features.dtype} {self.features.shape}")
        n = self.features.shape[0]
        # plain-ndarray view of the same mapping, one row per video: indexing a np.memmap builds a new memmap object per
        # access (3-4 us each, under the GIL), which was most of the time of a 512-row gather
        self._rows = np.asarray(self.features).reshape(n, -1)
        self.num_segments = int(self.meta["num_segments"])
        if num_dataload is None:
            self.order = np.arange(n, dtype=np.int64)
        else:
            reps, left = divmod(int(num_dataload), n)                       # dataset.py:70-75
            self.order = np.concatenate([np.tile(np.arange(n), reps), np.arange(left)]).astype(np.int64)
        self.labels = np.asarray(self.meta["labels"], dtype=np.int64)[self.order]

    def __len__(self):
        return int(self.order.shape[0])

    def __getitem__(self, index):
        row = int(self.order[index])
        return torch.from_numpy(np.array(self.features[row])), int(self.labels[index])

    def gather(self, indices: np.ndarray, out: torch.Tensor, out_labels: torch.Tensor) -> None:
        """Rows `indices` (dataset order) -> out[:len(indices)] / out_labels[:len(indices)] as ONE C-level row gather
        straight into the staging buffer (no intermediate tensors, no Python per row).  Measured on the build host, 512
        rows of 40 KB from the page cache: 3.0 ms (7 GB/s) for a Python loop of memmap row copies, 1.6 ms (13 GB/s) this
        way; more threads did not add bandwidth there."""
        rows = self.order[indices]                      # IndexError on a bad index; values are < n by construction
        k = int(rows.shape[0])
        dst = out.numpy().reshape(out.shape[0], -1)[:k]
        # mode='clip' selects numpy's unbuffered path when `out` is given ('raise' gathers into a temporary first: 3x
        # slower); nothing is ever clipped, the rows were validated by the lookup above
        np.take(self._rows, rows, axis=0, out=dst, mode='clip')
        out_labels.numpy()[:k] = self.labels[indices]


def paired_epoch_length(lengths: Sequence[int], batch_sizes: Sequence[int]) -> int:
    """Iterations of one paired epoch: zip stops with the shorter loader, each ending with one short batch."""
    return min(-(-int(n) // int(b)) for n, b in zip(lengths, batch_sizes))


def paired_epoch_plan(gen: torch.Generator, lengths: Sequence[int],
                      batch_sizes: Sequence[int]) -> Tuple[List[np.ndarray], int]:
    """The sampling decision of one epoch of main.py:343-346 (RandomSampler per domain, main.py:188, 199): one
    `torch.randperm` per dataset from `gen`, source first, and the epoch length.  Batch `it` of domain d is
    `epoch_batch(perms[d], it, batch_sizes[d])`.  Returns (perms, n_iter)."""
    perms = [torch.randperm(int(n), generator=gen).numpy() for n in lengths]
    return perms, paired_epoch_length(lengths, batch_sizes)


def epoch_batch(perm: np.ndarray, it: int, batch: int) -> np.ndarray:
    """Dataset positions of batch `it` (the last one of an epoch may be short)."""
    return perm[it * batch:(it + 1) * batch]


class PairedFeatureLoader:
    """`enumerate(zip(source_loader, target_loader))` of main.py:343-346 for two `PackedTSNDataSet`s: each epoch
    visits both sets in an independent random permutation (RandomSampler, main.py:188, 199), stops with the
    shorter one, and -- like DataLoader without drop_last -- ends with one short batch.  A background thread
    fills `depth` staging buffer sets (pinned when CUDA is present), so the caller only ever waits when the
    disk is slower than the GPU.

    Yields `((source_data, source_label), (target_data, target_label))`; the tensors are views of a staging
    buffer that stays untouched until TWO further batches have been requested (so an asynchronous H2D copy
    issued from it may still be in flight while the next batch is being consumed)."""

    def __init__(self, source: PackedTSNDataSet, target: PackedTSNDataSet, batch_sizes: Sequence[int],
                 seed: int = 0, depth: int = 3, pin_memory: Optional[bool] = None):
        if depth < 3:
            raise ValueError("depth must be >= 3 (current batch + previous batch + one being filled)")
        self.sets = (source, target)
        self.batch = (int(batch_sizes[0]), int(batch_sizes[1]))
        self.depth = depth
        self.gen = torch.Generator().manual_seed(seed)
        pin = torch.cuda.is_available() if pin_memory is None else bool(pin_memory)
        self.buffers = []
        for _ in range(depth):
            slot = []
            for ds, b in zip(self.sets, self.batch):
                x = torch.empty((b,) + tuple(ds.features.shape[1:]), dtype=torch.float32)
                y = torch.empty(b, dtype=torch.int64)
                slot.append((x.pin_memory(), y.pin_memory()) if pin else (x, y))
            self.buffers.append(slot)

    def __len__(self):
        return paired_epoch_length([len(ds) for ds in self.sets], self.batch)

    def __iter__(self) -> Iterator:
        perms, n_iter = paired_epoch_plan(self.gen, [len(ds) for ds in self.sets], self.batch)
        ready: "queue.Queue" = queue.Queue()
        free = threading.Semaphore(self.depth)       # staging slots the producer may still fill
        stop = threading.Event()

        def produce():
            try:
                for it in range(n_iter):
                    while not free.acquire(timeout=0.1):
                        if stop.is_set():
                            return
                    if stop.is_set():
                        return
                    slot = self.buffers[it % self.depth]
                    sizes = []
                    for d, (ds, b) in enumerate(zip(self.sets, self.batch)):
                        idx = epoch_batch(perms[d], it, b)
                        ds.gather(idx, slot[d][0], slot[d][1])
                        sizes.append(len(idx))
                    ready.put((it, sizes))
                ready.put(None)
            except BaseException as e:   # surface worker failures in the consumer
                ready.put(e)

        worker = threading.Thread(target=produce, daemon=True)
        worker.start()
        try:
            while True:
                item = ready.get()
                if item is None:
                    return
                if isinstance(item, BaseException):
                    raise item
                it, sizes = item
                slot = self.buffers[it % self.depth]
                yield tuple((slot[d][0][:sizes[d]], slot[d][1][:sizes[d]]) for d in range(2))
                if it >= 1:
                    free.release()               # batch it-1 is no longer referenced: its slot may be refilled
        finally:
            stop.set()
            worker.join(timeout=5)


# ---- device-resident shards ------------------------------------------------------------------------------
class DeviceFeatureBank:
    """The rows of a `PackedTSNDataSet` in device memory, uploaded once: `features` is `(videos, T*feat_dim)` fp32 on
    `device` (each distinct video once; `order` maps dataset positions -- num_dataload replication -- to rows, and
    `labels` is in dataset order, as in the dataset).  The shard streams through ONE pinned staging buffer of
    `chunk_bytes` (two halves, so that reading the next chunk overlaps the copy of the last); the memmap is never
    pinned as a whole.  Before allocating, free device memory must cover the bank plus `headroom_bytes` (what the
    training step and the rest of the process still need), otherwise `Ta3nError`."""

    def __init__(self, dataset: PackedTSNDataSet, device=None, chunk_bytes: int = 64 << 20,
                 headroom_bytes: int = 2 << 30):
        from ._lib import Ta3nError
        dev = torch.device(device if device is not None else "cuda")
        if dev.type != "cuda":
            raise Ta3nError("DeviceFeatureBank needs a CUDA device")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        src = dataset._rows
        n, row_floats = int(src.shape[0]), int(src.shape[1])
        if row_floats % 4:
            raise Ta3nError(f"rows of {row_floats} floats are not 16-byte multiples; the device gather needs them")
        nbytes = n * row_floats * 4
        free, _ = torch.cuda.mem_get_info(dev)
        cached = torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)   # this process may reuse it
        if nbytes + int(headroom_bytes) > free + cached:
            raise Ta3nError(f"feature bank of {nbytes / 2**30:.2f} GiB ({n} videos x {row_floats} floats) does not fit "
                            f"on {dev}: {(free + cached) / 2**30:.2f} GiB free, {int(headroom_bytes) / 2**30:.2f} GiB "
                            "kept for training; use the host pipeline (PairedFeatureLoader) for this dataset")
        self.device = dev
        self.row_shape = tuple(int(s) for s in dataset.features.shape[1:])
        self.order = dataset.order
        self.labels = dataset.labels
        self.features = torch.empty((n, row_floats), device=dev, dtype=torch.float32)
        per = max(1, int(chunk_bytes) // (2 * row_floats * 4))          # rows per half of the staging buffer
        stage = torch.empty((2, per, row_floats), dtype=torch.float32, pin_memory=True)
        done = [None, None]
        with torch.cuda.device(dev):
            for k, a in enumerate(range(0, n, per)):
                h, b = k % 2, min(n, a + per)
                if done[h] is not None:
                    done[h].synchronize()               # the copy out of this half has finished
                np.copyto(stage[h].numpy()[:b - a], src[a:b])
                self.features[a:b].copy_(stage[h][:b - a], non_blocking=True)
                done[h] = torch.cuda.Event()
                done[h].record()
            torch.cuda.current_stream().synchronize()

    def __len__(self):
        return int(self.order.shape[0])

    @property
    def nbytes(self) -> int:
        return self.features.numel() * 4


class DevicePairedSampler:
    """`PairedFeatureLoader(source, target, batch_sizes, seed)` over two `DeviceFeatureBank`s: the same epochs (the
    same `paired_epoch_plan`, one generator seeded once), but the batches are gathered on the device by the first
    launch of the captured step that the sampler is handed to (`TrainStep(..., sampler=...)`, C ABI
    `ta3n_gather_batch`).  `start_epoch()` draws the next epoch, uploads its row and label lists (outside the
    graph, on the current stream), rewinds the device iteration index and returns the number of iterations; each
    `TrainStep.run()` then consumes one of them."""

    def __init__(self, source: DeviceFeatureBank, target: DeviceFeatureBank, batch_sizes: Sequence[int],
                 seed: int = 0):
        if source.device != target.device:
            raise ValueError("both banks must live on the same device")
        if source.row_shape != target.row_shape:
            raise ValueError(f"source rows {source.row_shape} and target rows {target.row_shape} differ")
        self.banks = (source, target)
        self.batch = (int(batch_sizes[0]), int(batch_sizes[1]))
        if min(self.batch) < 1:
            raise ValueError("batch sizes must be >= 1")
        self.device = source.device
        self.row_shape = source.row_shape
        self.lengths = (len(source), len(target))
        self.gen = torch.Generator().manual_seed(seed)
        dev = self.device
        # fixed addresses, captured by the step's graph; zeros until the first epoch
        self.rows = [torch.zeros(n, device=dev, dtype=torch.int32) for n in self.lengths]
        self.labels = torch.zeros(self.lengths[0], device=dev, dtype=torch.int64)
        self.state = torch.zeros(2, device=dev, dtype=torch.int32)      # {iteration, arrival counter}
        # the target label list: only a step that trains on the target labels (use_target='Sv') asks for it
        self.labels_t = None
        self._perm_t = None
        self.n_iter = 0        # iterations of the current epoch (0 before the first start_epoch)
        self.issued = 0        # of which run() has consumed

    def __len__(self):
        return paired_epoch_length(self.lengths, self.batch)

    def start_epoch(self) -> int:
        perms, n_iter = paired_epoch_plan(self.gen, self.lengths, self.batch)
        for d, bank in enumerate(self.banks):
            self.rows[d].copy_(torch.from_numpy(bank.order[perms[d]].astype(np.int32)))
        self.labels.copy_(torch.from_numpy(self.banks[0].labels[perms[0]]))
        self._perm_t = perms[1]
        if self.labels_t is not None:
            self.labels_t.copy_(torch.from_numpy(self.banks[1].labels[perms[1]]))
        self.rewind()
        self.n_iter = n_iter
        return n_iter

    def enable_target_labels(self) -> None:
        """Keep the target label list on the device too, so that ``enqueue_gather`` can fill the target slot labels
        (``TrainStep(use_target='Sv')``); the current epoch's list is uploaded at once.  Idempotent."""
        if self.labels_t is None:
            self.labels_t = torch.zeros(self.lengths[1], device=self.device, dtype=torch.int64)
            if self._perm_t is not None:
                self.labels_t.copy_(torch.from_numpy(self.banks[1].labels[self._perm_t]))

    def rewind(self) -> None:
        """Restart the current epoch at iteration 0 (current stream)."""
        self.state.zero_()
        self.issued = 0

    def take(self) -> None:
        """Account for one more iteration of the epoch; raises past its end (host-side, before anything runs)."""
        if self.issued >= self.n_iter:
            raise RuntimeError(f"the epoch has {self.n_iter} iterations and all have run; call start_epoch()"
                               if self.n_iter else "call start_epoch() before the first run()")
        self.issued += 1

    def enqueue_gather(self, xs: torch.Tensor, xt: torch.Tensor, labels: torch.Tensor, valid: torch.Tensor,
                       stream: int, labels_t: Optional[torch.Tensor] = None) -> None:
        """Fill one input slot (source / target features, source labels, {real source rows, real target rows})
        with the current iteration's batch and advance the device iteration index: one launch.  ``labels_t``: the
        slot's target labels, filled too (``ta3n_gather_batch_labelled``; needs ``enable_target_labels()``)."""
        from . import _lib
        (bs, bt), (s, t) = self.batch, self.banks
        if (xs.shape[0], xt.shape[0]) != (bs, bt) or tuple(xs.shape[1:]) != self.row_shape or \
                tuple(xt.shape[1:]) != self.row_shape:
            raise ValueError(f"slot {tuple(xs.shape)} + {tuple(xt.shape)} does not match the sampler's batches "
                             f"{bs} + {bt} of {self.row_shape}")
        if labels_t is not None:
            if self.labels_t is None:
                raise ValueError("target slot labels need enable_target_labels()")
            _lib.check(_lib.load().ta3n_gather_batch_labelled(
                s.features.data_ptr(), s.features.shape[0], self.rows[0].data_ptr(), self.labels.data_ptr(),
                self.lengths[0], bs, xs.data_ptr(), labels.data_ptr(),
                t.features.data_ptr(), t.features.shape[0], self.rows[1].data_ptr(), self.labels_t.data_ptr(),
                self.lengths[1], bt, xt.data_ptr(), labels_t.data_ptr(),
                s.features.shape[1], valid.data_ptr(), self.state.data_ptr(), stream))
            return
        _lib.check(_lib.load().ta3n_gather_batch(
            s.features.data_ptr(), s.features.shape[0], self.rows[0].data_ptr(), self.labels.data_ptr(),
            self.lengths[0], bs, xs.data_ptr(), labels.data_ptr(),
            t.features.data_ptr(), t.features.shape[0], self.rows[1].data_ptr(), self.lengths[1], bt, xt.data_ptr(),
            s.features.shape[1], valid.data_ptr(), self.state.data_ptr(), stream))


class DeviceEvalSampler:
    """The validation loader of main.py:176-178 (`shuffle=False`, `batch_size[2]`) over one `DeviceFeatureBank`: the
    dataset positions in order, `ceil(N / batch)` batches, the last one short.  Each batch is gathered on the device
    by the first launch of the captured validation step (`EvalStep(..., sampler=...)`, C ABI `ta3n_gather_rows`).
    `start_epoch()` uploads the row list once (`bank.order`: the num_dataload tiling) and rewinds; each
    `EvalStep` replay then consumes one batch."""

    def __init__(self, bank: DeviceFeatureBank, batch: int):
        if int(batch) < 1:
            raise ValueError("batch size must be >= 1")
        self.bank = bank
        self.batch = int(batch)
        self.device = bank.device
        self.row_shape = bank.row_shape
        self.n = len(bank)
        dev = self.device
        # fixed addresses, captured by the step's graph
        self.rows = torch.zeros(self.n, device=dev, dtype=torch.int32)
        self.labels = torch.zeros(self.n, device=dev, dtype=torch.int64)
        self.state = torch.zeros(2, device=dev, dtype=torch.int32)      # {batch index, arrival counter}
        self.uploaded = False
        self.n_iter = 0
        self.issued = 0

    def __len__(self):
        return -(-self.n // self.batch)

    def start_epoch(self) -> int:
        if not self.uploaded:
            self.rows.copy_(torch.from_numpy(self.bank.order.astype(np.int32)))
            self.labels.copy_(torch.from_numpy(np.ascontiguousarray(self.bank.labels, dtype=np.int64)))
            self.uploaded = True
        self.rewind()
        self.n_iter = len(self)
        return self.n_iter

    def rewind(self) -> None:
        """Restart the epoch at batch 0 (current stream)."""
        self.state.zero_()
        self.issued = 0

    def take(self) -> None:
        """Account for one more batch of the epoch; raises past its end (host-side, before anything runs)."""
        if self.issued >= self.n_iter:
            raise RuntimeError(f"the epoch has {self.n_iter} batches and all have run; call start_epoch()"
                               if self.n_iter else "call start_epoch() before the first run")
        self.issued += 1

    def enqueue_gather(self, x: torch.Tensor, labels: torch.Tensor, valid: torch.Tensor, stream: int) -> None:
        """Fill the input slot (features, labels, {real rows}) with the current batch and advance the device batch
        index: one launch."""
        from . import _lib
        if x.shape[0] != self.batch or tuple(x.shape[1:]) != self.row_shape:
            raise ValueError(f"slot {tuple(x.shape)} does not match the sampler's batches of {self.batch} x "
                             f"{self.row_shape}")
        f = self.bank.features
        _lib.check(_lib.load().ta3n_gather_rows(
            f.data_ptr(), f.shape[0], self.rows.data_ptr(), self.labels.data_ptr(), self.n, self.batch, x.data_ptr(),
            labels.data_ptr(), f.shape[1], valid.data_ptr(), self.state.data_ptr(), stream))


def _main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description="Pack the frames a list file's clips contribute into one .npy shard")
    ap.add_argument("list_file")
    ap.add_argument("out_path")
    ap.add_argument("--num_segments", type=int, default=5)
    ap.add_argument("--new_length", type=int, default=1)
    ap.add_argument("--modality", default="RGB")
    ap.add_argument("--image_tmpl", default="img_{:05d}.t7")
    ap.add_argument("--rule", default="test", choices=["test", "val"])
    a = ap.parse_args(argv)
    shape = pack_list(a.list_file, a.out_path, a.num_segments, a.new_length, a.modality, a.image_tmpl, a.rule)
    print(f"{a.out_path}: {shape} float32, {np.prod(shape) * 4 / 1e6:.1f} MB")


if __name__ == "__main__":
    _main()
