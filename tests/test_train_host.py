"""Host-side logic of ta3n_b200.train that needs no GPU: flat-buffer layout, parameter flattening, schedules."""
import pytest
import torch

from oracle import ta3n_oracle as orc
from ta3n_b200 import Ta3nError
from ta3n_b200 import train as T
from ta3n_b200.models import VideoModel


def _model(C=5):
    torch.manual_seed(3)
    return VideoModel(C, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=512, partial_bn=False,
                      verbose=False)


def test_bucket_layout_is_backward_completion_order_with_aligned_slots():
    params = _model().path_parameters()
    order, offs, total, early = T.bucket_layout(params)
    assert order == list(range(6, len(params))) + list(range(6))      # shared layer + frame discriminator last
    assert sorted(order) == list(range(len(params)))
    end = 0
    for idx in order:
        assert offs[idx] % 64 == 0 and offs[idx] >= end                # 256-byte aligned, no overlap
        end = offs[idx] + params[idx].numel()
        if idx == len(params) - 1:
            assert early == -(-end // 64) * 64                         # early bucket ends after the last video-head tensor
    assert total >= end and total % 64 == 0
    # C=5 makes the class-head bias 5 floats: the slot after it must still be aligned
    sizes = sorted(p.numel() for p in params)
    assert 5 in sizes and 2 in sizes


def test_flatten_parameters_preserves_values_names_and_is_idempotent():
    model = _model()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    flat = T.flatten_parameters(model)
    assert T.flatten_parameters(model) is flat                         # idempotent: same buffer
    after = model.state_dict()
    assert list(after.keys()) == list(before.keys())
    for k in before:
        assert torch.equal(after[k], before[k]), k
    params = model.path_parameters()
    _, offs, total, _ = T.bucket_layout(params)
    assert flat.numel() == total
    for i, p in enumerate(params):
        assert p.data_ptr() == flat.data_ptr() + 4 * offs[i]
    # writes through the flat buffer are writes to the parameters (the optimizer kernel relies on this) ...
    flat.zero_()
    assert all(float(p.detach().abs().sum()) == 0.0 for p in params)
    # ... parameters the path never uses stay outside the flat buffer and keep their values
    assert torch.equal(model.fc_feature_source.weight, before["fc_feature_source.weight"])
    # load_state_dict copies in place: the views survive a checkpoint load
    model.load_state_dict(before)
    assert all(p.data_ptr() == flat.data_ptr() + 4 * offs[i] for i, p in enumerate(params))
    assert torch.equal(model.state_dict()["fc_feature_shared_source.weight"], before["fc_feature_shared_source.weight"])


@pytest.mark.parametrize("frame_attn,kw,exc,match", [
    ("TransAttn", dict(mode="phased"), NotImplementedError, "use_attn_frame"),
    ("none", dict(mode="legacy", class_weight=torch.ones(5)), ValueError, "class_weight needs mode='phased'"),
    ("none", dict(mode="legacy", beta=(-1.0, 0.6, 0.5)), ValueError, "negative beta"),
    ("none", dict(mode="legacy", domain_weight=(1.0, 0.5)), ValueError, "domain_weight needs mode='phased'"),
    # frame attention selects the per-operator sequence, which has no domain weights either
    ("TransAttn", dict(domain_weight=(1.0, 0.5)), ValueError, "domain_weight needs mode='phased'"),
])
def test_executor_refusals_come_before_the_device_check(monkeypatch, frame_attn, kw, exc, match):
    monkeypatch.delenv("TA3N_STEP_MODE", raising=False)
    torch.manual_seed(3)
    m = VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, use_attn_frame=frame_attn,
                   verbose=False).train()
    kw = dict(dict(beta=(0.75, 0.6, 0.5)), **kw)
    with pytest.raises(exc, match=match):
        T.TrainStep(m, 4, 4, **kw)
    # the step program takes the weights: that configuration passes every check and stops at the device
    if frame_attn == "none":
        with pytest.raises(Ta3nError, match="CUDA"):
            T.TrainStep(m, 4, 4, **dict(kw, mode="phased"))


def test_learning_rate_schedule_matches_oracle_restatement_of_main_py():
    for p in (0.0, 0.1, 0.5, 1.0):
        assert T.lr_dann(3e-2, p) == orc.lr_dann(3e-2, p)              # main.py:800-802
    assert T.lr_dann(3e-2, 0.0) == 3e-2
    cfg = T.SGDNesterov(lr=3e-2)
    assert (cfg.momentum, cfg.weight_decay, cfg.clip_gradient) == (0.9, 1e-4, 20.0)   # opts.py defaults


def test_loss_helpers_match_the_oracle_statements():
    """ta3n_b200.loss (torch-op heads next to the path, loss.py:8-30) against the oracle's restatements, which are
    pinned to the live reference in tests/test_oracle_vs_reference.py."""
    import torch

    from oracle import ta3n_oracle as orc
    from ta3n_b200 import loss as L
    g = torch.Generator().manual_seed(3)
    a, b = torch.randn(11, 7, generator=g), torch.randn(11, 7, generator=g)
    d = torch.randn(11, 2, generator=g)
    assert torch.allclose(L.dis_MCD(a, b), orc.dis_MCD(a, b), rtol=0, atol=1e-7)
    assert torch.allclose(L.attentive_entropy(a, d), orc.attentive_entropy(a, d), rtol=0, atol=1e-6)
    assert float(L.dis_MCD(a, a)) == 0.0
