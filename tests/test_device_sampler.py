"""Device-resident input pipeline: feature banks in device memory, each paired mini-batch gathered by the first launch
of the captured step (ta3n_gather_batch, dataset.DeviceFeatureBank / DevicePairedSampler, TrainStep(sampler=...)).

CPU: the shared epoch plan against what PairedFeatureLoader yields, the C ABI's argument checks, what TrainStep
refuses.  GPU: the gather kernel alone in a replayed graph over whole epochs (and on a bank above 2^31 floats), and
TrainStep fed by the sampler against TrainStep fed the same batches through load(), bit for bit.
"""
import copy
import json
import os
import types

import numpy as np
import pytest
import torch

from ta3n_b200 import dataset as D

gpu = pytest.mark.gpu


def _shard(root, name, n, T, F, seed, num_dataload=None, n_class=5):
    """A packed shard as pack_list writes it (fp32 (n, T, F) .npy + .json with the labels)."""
    rng = np.random.default_rng(seed)
    path = os.path.join(str(root), name + ".npy")
    np.save(path, rng.standard_normal((n, T, F), dtype=np.float32))
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, n_class, n)]}, f)
    return D.PackedTSNDataSet(path, num_dataload=num_dataload)


# (videos, num_dataload) per domain, batch sizes
PLAN_CASES = {
    "unequal_lengths_both_short": (((9, 9), (5, 7)), (4, 3)),       # 3 iterations, ends 1 + 1
    "short_source_only": (((10, None), (9, None)), (4, 3)),         # 3 iterations, ends 2 + 3
    "short_target_only": (((12, None), (8, None)), (4, 3)),         # 3 iterations, ends 4 + 2
    "num_dataload_not_n": (((7, 11), (5, 13)), (4, 6)),             # tiled lists; target has more batches
}


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_epoch_plan_equals_paired_loader(tmp_path, case):
    """paired_epoch_plan (the decision both paths draw from) against the batches PairedFeatureLoader yields, batch
    for batch over 3 epochs, and both against the loader's original rule (one randperm per set, source first)."""
    (src, tgt), batch = PLAN_CASES[case]
    sets = (_shard(tmp_path, "s", src[0], 3, 8, 1, src[1]), _shard(tmp_path, "t", tgt[0], 3, 8, 2, tgt[1]))
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch_sizes=batch, seed=11, pin_memory=False)
    gen, old = torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)
    lengths = [len(s) for s in sets]
    for epoch in range(3):
        perms, n_iter = D.paired_epoch_plan(gen, lengths, batch)
        old_perms = [torch.randperm(n, generator=old).numpy() for n in lengths]
        assert all(np.array_equal(a, b) for a, b in zip(perms, old_perms))
        assert n_iter == len(loader) == min(-(-n // b) for n, b in zip(lengths, batch))
        got = list(loader)
        assert len(got) == n_iter
        for it, pair in enumerate(got):
            for d in range(2):
                idx = D.epoch_batch(perms[d], it, batch[d])
                np.testing.assert_array_equal(idx, old_perms[d][it * batch[d]:(it + 1) * batch[d]])
                x, y = pair[d]
                want = np.stack([sets[d][int(i)][0].numpy() for i in idx])
                assert np.array_equal(x.numpy(), want), (case, epoch, it, d)
                assert np.array_equal(y.numpy(), sets[d].labels[idx]), (case, epoch, it, d)
        sizes = [(p[0][0].shape[0], p[1][0].shape[0]) for p in got]
        assert all(s[0] >= 1 and s[1] >= 1 for s in sizes)


def test_gather_entry_validates_arguments_without_gpu():
    from ta3n_b200 import _lib
    lib = _lib.load()
    g = lib.ta3n_gather_batch
    # bank_s, n_rows_s, rows_s, labels_s, n_epoch_s, batch_s, x_s, y_s, bank_t, n_rows_t, rows_t, n_epoch_t, batch_t,
    # x_t, row_floats, valid_rows, state, stream
    ok = [256, 10, 512, 768, 10, 4, 1024, 1280, 1536, 8, 1792, 8, 3, 2048, 40, 2304, 2560, None]

    def call(**kw):
        names = ["bank_s", "n_rows_s", "rows_s", "labels_s", "n_epoch_s", "batch_s", "x_s", "y_s", "bank_t",
                 "n_rows_t", "rows_t", "n_epoch_t", "batch_t", "x_t", "row_floats", "valid", "state", "stream"]
        args = dict(zip(names, ok))
        args.update(kw)
        return g(*[args[n] for n in names])

    for kw, msg in ((dict(bank_s=None), b"null source"), (dict(labels_s=None), b"null source"),
                    (dict(x_t=None), b"null target"), (dict(state=None), b"null valid_rows / state"),
                    (dict(valid=None), b"null valid_rows / state"), (dict(batch_s=0), b"batch sizes"),
                    (dict(batch_t=0), b"batch sizes"), (dict(batch_s=60000, batch_t=6000), b"batch sizes"),
                    (dict(row_floats=42), b"multiple of 4"), (dict(row_floats=0), b"multiple of 4"),
                    (dict(n_epoch_t=0), b"empty epoch"), (dict(n_rows_s=1 << 31), b"2^31"),
                    (dict(bank_s=260), b"16-byte aligned"), (dict(x_t=2052), b"16-byte aligned"),
                    (dict(n_rows_t=1 << 30, row_floats=1 << 40), b"too large")):
        assert call(**kw) == 1, kw
        err = lib.ta3n_last_error()
        assert b"ta3n_gather_batch" in err and msg in err, (kw, err)


def _cpu_model():
    from ta3n_b200.models import VideoModel
    return VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, verbose=False).train()


def test_train_step_refuses_sampler_with_double_buffer_or_several_ranks(monkeypatch):
    from ta3n_b200 import train
    fake = types.SimpleNamespace(batch=(4, 4))
    with pytest.raises(ValueError, match="double_buffer"):
        train.TrainStep(_cpu_model(), 4, 4, beta=[0.75, 0.75, 0.5], sampler=fake, double_buffer=True)
    with pytest.raises(ValueError, match="sampler batches"):
        train.TrainStep(_cpu_model(), 4, 3, beta=[0.75, 0.75, 0.5], sampler=fake)
    monkeypatch.setattr(train.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(train.dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(NotImplementedError, match="single rank"):
        train.TrainStep(_cpu_model(), 4, 4, beta=[0.75, 0.75, 0.5], sampler=fake)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _banks(tmp_path, T, F, src, tgt, batch, seed=3):
    sets = (_shard(tmp_path, "s", src[0], T, F, seed, src[1]), _shard(tmp_path, "t", tgt[0], T, F, seed + 1, tgt[1]))
    banks = tuple(D.DeviceFeatureBank(s, chunk_bytes=T * F * 4 * 6) for s in sets)      # several staging chunks
    return sets, banks


@gpu
@pytest.mark.parametrize("F", [64, 2048])
def test_gather_kernel_in_a_replayed_graph_matches_the_loader(tmp_path, F):
    """The gather alone, captured once and replayed over two whole epochs: every slot bit-equal to index_select of
    the bank at the loader's batch, padded rows zero, labels and the {real rows} pair right, the index advancing
    once per replay.  F = 2048 rows span three 16 KB chunks (the last one partial)."""
    from ta3n_b200 import _lib
    T, batch = 5, (8, 5)
    sets, banks = _banks(tmp_path, T, F, (37, 41), (23, None), batch)
    for s, b in zip(sets, banks):
        assert torch.equal(b.features.cpu(), torch.from_numpy(np.array(s._rows)))
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=7)
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=7, pin_memory=False)
    dev = banks[0].device
    xs = torch.full((batch[0], T, F), float("nan"), device=dev)
    xt = torch.full((batch[1], T, F), float("nan"), device=dev)
    lab = torch.full((batch[0],), -5, device=dev, dtype=torch.int64)
    valid = torch.zeros(2, device=dev, dtype=torch.int32)
    assert sampler.start_epoch() == len(loader) == 5
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sampler.enqueue_gather(xs, xt, lab, valid, torch.cuda.current_stream().cuda_stream)
    for epoch in range(2):
        if epoch:
            assert sampler.start_epoch() == 5
        for it, ((hx_s, hy_s), (hx_t, _)) in enumerate(loader):
            g.replay()
            torch.cuda.synchronize()
            assert sampler.state.tolist() == [it + 1, 0]
            ns, nt = hx_s.shape[0], hx_t.shape[0]
            assert valid.tolist() == [ns, nt]
            for x, hx, d, n in ((xs, hx_s, 0, ns), (xt, hx_t, 1, nt)):
                assert torch.equal(x[:n].cpu(), hx), (epoch, it, d)
                assert torch.equal(x[n:].cpu(), torch.zeros_like(x[n:].cpu())), (epoch, it, d)
            rows = sampler.rows[0][it * batch[0]:it * batch[0] + ns].long()
            assert torch.equal(xs[:ns].reshape(ns, -1), banks[0].features.index_select(0, rows))
            assert torch.equal(lab[:ns].cpu(), hy_s) and torch.all(lab[ns:] == 0)
        assert (ns, nt) == (8, 3)           # 41 source positions (37 videos tiled), 23 target
    # the launch is counted and reported under its own label
    _lib.timing_enable(True)
    n0 = _lib.launch_count()
    sampler.rewind()
    sampler.enqueue_gather(xs, xt, lab, valid, torch.cuda.current_stream().cuda_stream)
    assert _lib.launch_count() == n0 + 1
    rep = _lib.timing_report()
    _lib.timing_enable(False)
    assert rep["gather_batch"][0] == 1


@gpu
def test_gather_from_a_bank_above_2_31_floats():
    """64-bit offsets: rows past float index 2^31 (byte offset 2^33) of an 8.6 GB bank, straight through the C ABI."""
    from ta3n_b200 import _lib
    row_floats = 5 * 2048
    n_rows = (1 << 31) // row_floats + 64
    need = n_rows * row_floats * 4
    free, _ = torch.cuda.mem_get_info()
    if free < need + (4 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB + 4 GiB free, {free / 2**30:.1f} GiB free")
    dev = torch.device("cuda")
    bank = torch.empty(n_rows, row_floats, device=dev)
    pick = torch.tensor([n_rows - 1, 0, n_rows - 40, (1 << 31) // row_floats + 3, n_rows // 2, n_rows - 2],
                        device=dev)
    bank[pick] = torch.randn(pick.numel(), row_floats, device=dev)
    rows, rows_t = pick.to(torch.int32), pick.flip(0).to(torch.int32)
    labels = torch.arange(pick.numel(), device=dev, dtype=torch.int64) + 10
    xs, xt = torch.empty(4, row_floats, device=dev), torch.empty(3, row_floats, device=dev)
    ys, valid = torch.empty(4, device=dev, dtype=torch.int64), torch.empty(2, device=dev, dtype=torch.int32)
    state = torch.zeros(2, device=dev, dtype=torch.int32)
    st = torch.cuda.current_stream().cuda_stream
    for it in range(2):         # source positions [0, 4) then [4, 6) + 2 padded rows; target [0, 3) then [3, 5)
        _lib.check(_lib.load().ta3n_gather_batch(bank.data_ptr(), n_rows, rows.data_ptr(), labels.data_ptr(), 6, 4,
                                                 xs.data_ptr(), ys.data_ptr(), bank.data_ptr(), n_rows,
                                                 rows_t.data_ptr(), 5, 3, xt.data_ptr(),
                                                 row_floats, valid.data_ptr(), state.data_ptr(), st))
        torch.cuda.synchronize()
        ns, nt = min(4, 6 - 4 * it), min(3, 5 - 3 * it)
        assert valid.tolist() == [ns, nt] and state.tolist() == [it + 1, 0]
        assert torch.equal(xs[:ns], bank.index_select(0, pick[4 * it:4 * it + ns]))
        assert torch.equal(xt[:nt], bank.index_select(0, pick.flip(0)[3 * it:3 * it + nt]))
        assert torch.all(xs[ns:] == 0) and torch.all(xt[nt:] == 0)
        assert torch.equal(ys[:ns], labels[4 * it:4 * it + ns]) and torch.all(ys[ns:] == 0)
    del bank
    torch.cuda.empty_cache()


@gpu
def test_gather_turns_a_row_id_outside_the_bank_into_a_nan_row():
    """A broken row list passed through the C ABI never reads outside the bank: that slot row is NaN, the rest exact."""
    from ta3n_b200 import _lib
    dev = torch.device("cuda")
    bank = torch.randn(6, 40, device=dev)
    rows = torch.tensor([2, 6, -1, 5], device=dev, dtype=torch.int32)
    labels = torch.arange(4, device=dev, dtype=torch.int64)
    xs, xt = torch.zeros(4, 40, device=dev), torch.zeros(2, 40, device=dev)
    ys, valid = torch.zeros(4, device=dev, dtype=torch.int64), torch.zeros(2, device=dev, dtype=torch.int32)
    state = torch.zeros(2, device=dev, dtype=torch.int32)
    _lib.check(_lib.load().ta3n_gather_batch(bank.data_ptr(), 6, rows.data_ptr(), labels.data_ptr(), 4, 4,
                                             xs.data_ptr(), ys.data_ptr(), bank.data_ptr(), 6, rows.data_ptr(), 2, 2,
                                             xt.data_ptr(), 40, valid.data_ptr(), state.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(xs[0], bank[2]) and torch.equal(xs[3], bank[5]) and torch.equal(xt[0], bank[2])
    assert torch.isnan(xs[1]).all() and torch.isnan(xs[2]).all() and torch.isnan(xt[1]).all()
    assert valid.tolist() == [4, 2] and state.tolist() == [1, 0] and torch.equal(ys, labels)


@gpu
def test_bank_refuses_what_does_not_fit(tmp_path):
    from ta3n_b200 import Ta3nError
    s = _shard(tmp_path, "s", 4, 5, 16, 0)
    with pytest.raises(Ta3nError, match="does not fit"):
        D.DeviceFeatureBank(s, headroom_bytes=1 << 50)


def _gpu_model(mcd):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(0)
    kw = dict(ens_DA="MCD") if mcd else {}
    return VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=96, verbose=False,
                      **kw).cuda().train()


@gpu
@pytest.mark.parametrize("mode", ["legacy", "phased", "mcd", "legacy_eager"])
def test_train_step_from_device_sampler_is_bit_identical_to_load(tmp_path, mode):
    """TrainStep fed by the device sampler against TrainStep fed the same batches through load(), seeded alike, over
    two epochs with short last batches on both sides: loss, every parameter and every momentum value equal bit for
    bit after every step (the slot is zeroed before a short load(), so that the inputs are byte-identical)."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    T, batch = 5, (8, 6)
    sets, banks = _banks(tmp_path, T, 2048, (21, None), (9, 14), batch)        # 3 iterations, ends 5 + 2
    model_a = _gpu_model(mode == "mcd")
    model_b = copy.deepcopy(model_a)
    kw = dict(beta=[0.75, 0.75, 0.5], optimizer=SGDNesterov(lr=0.01), seed=123,
              mode="phased" if mode == "phased" else "legacy", use_graph=mode != "legacy_eager",
              mu=0.7 if mode == "mcd" else 0.0)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    step_a = TrainStep(model_a, *batch, sampler=sampler, **{**kw, "optimizer": SGDNesterov(lr=0.01)})
    step_b = TrainStep(model_b, *batch, **kw)
    if mode != "legacy_eager":
        assert step_a.launches_per_step == step_b.launches_per_step + 1
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=4)
    n_step = 0
    for epoch in range(2):
        assert sampler.start_epoch() == len(loader) == 3
        for (xs, ys), (xt, _) in loader:
            if xs.shape[0] < batch[0] or xt.shape[0] < batch[1]:
                step_b.xs.zero_(), step_b.xt.zero_(), step_b.labels.zero_()
            step_b.load(xs, xt, ys)
            loss_b = step_b.run().clone()
            loss_a = step_a.run().clone()
            torch.cuda.synchronize()
            n_step += 1
            assert torch.equal(step_a.xs, step_b.xs) and torch.equal(step_a.xt, step_b.xt)
            assert torch.equal(step_a.valid, step_b.valid) and torch.equal(step_a.labels, step_b.labels)
            assert torch.equal(loss_a, loss_b), (epoch, n_step, loss_a.item(), loss_b.item())
            assert torch.isfinite(loss_a).all()
            assert torch.equal(step_a.flat_param, step_b.flat_param), (epoch, n_step)
            assert torch.equal(step_a.momentum_buf, step_b.momentum_buf), (epoch, n_step)
        assert step_a.valid.tolist() == [5, 2]
        with pytest.raises(RuntimeError, match="start_epoch"):
            step_a.run()                     # past the end of the epoch: refused on the host
    assert n_step == 6
    with pytest.raises(RuntimeError, match="device sampler"):
        step_a.load(xs, xt, ys)
    with pytest.raises(RuntimeError, match="device sampler"):
        step_a(xs, xt, ys)
    with pytest.raises(RuntimeError, match="device sampler"):
        step_a.prefetch(xs, xt, ys)


@gpu
def test_train_step_with_sampler_refusals(tmp_path):
    from ta3n_b200.train import TrainStep
    _, banks = _banks(tmp_path, 5, 2048, (6, None), (5, None), (4, 4))
    sampler = D.DevicePairedSampler(banks[0], banks[1], (4, 4), seed=0)
    with pytest.raises(ValueError, match="double_buffer"):
        TrainStep(_gpu_model(False), 4, 4, beta=[0.75, 0.75, 0.5], sampler=sampler, double_buffer=True)
    step = TrainStep(_gpu_model(False), 4, 4, beta=[0.75, 0.75, 0.5], sampler=sampler)
    with pytest.raises(RuntimeError, match="before the first run"):
        step.run()
    assert sampler.start_epoch() == 2
    step.run(), step.run()
    with pytest.raises(RuntimeError, match="all have run"):
        step.run()
