"""The C-ABI shared library loads and exports every symbol include/ta3n_b200.h declares (no compute)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "ta3n_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ta3n_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from ta3n_b200 import build
    build.build()                       # nvcc cross-compiles sm_90a without a GPU
    from ta3n_b200 import _lib
    return _lib.load()


def test_header_and_binding_agree(lib):
    from ta3n_b200 import _lib
    names = declared_functions()
    assert len(names) >= 20
    assert sorted(_lib.SIGNATURES) == names


def test_every_declared_symbol_is_exported(lib):
    raw = ctypes.CDLL(lib._name)
    for name in declared_functions():
        assert hasattr(raw, name), f"{name} declared in the header but not exported"


def test_abi_version_matches_header(lib):
    """The library, the header and the binding agree on the ABI version (bumped whenever a symbol goes)."""
    from ta3n_b200 import _lib
    header = int(re.search(r"#define\s+TA3N_ABI_VERSION\s+(\d+)", open(HEADER).read()).group(1))
    assert lib.ta3n_abi_version() == header == _lib.ABI_VERSION


def test_engine_switch(lib):
    from ta3n_b200 import _lib
    assert _lib.get_gemm_engine() == "tf32x3"          # the library default: the parity-tested product engine
    _lib.set_gemm_engine("tf32")
    assert _lib.get_gemm_engine() == "tf32"
    _lib.set_gemm_engine("fp32")
    assert _lib.get_gemm_engine() == "fp32"
    assert lib.ta3n_set_gemm_engine(7) != 0
    assert b"unknown GEMM engine" in lib.ta3n_last_error()
    _lib.set_gemm_engine("tf32x3")          # the library default


def test_argument_validation_needs_no_gpu(lib):
    # null pointers / bad sizes are rejected on the host before any CUDA call
    rc = lib.ta3n_disc_fwd(None, 4, 8, 8, None, None, None, None, None, None, None)
    assert rc == 1
    assert b"ta3n_disc_fwd" in lib.ta3n_last_error()
    rc = lib.ta3n_gemm_tn(None, None, None, 0, 0, 0, None)
    assert rc == 1
    # optimizer entry: null buffers, then buffers that are not 16-byte aligned
    assert lib.ta3n_sgd_nesterov_step(None, None, None, 10, None, 0.9, 1e-4, 20.0, None, 0, None, None) == 1
    assert lib.ta3n_sgd_nesterov_step(4, 16, 32, 10, 64, 0.9, 1e-4, 0.0, None, 0, None, None) == 1
    assert b"16-byte aligned" in lib.ta3n_last_error()
    assert lib.ta3n_sgd_nesterov_step(16, 32, 48, 10, 64, -0.1, 1e-4, 0.0, None, 0, None, None) == 1
    assert lib.ta3n_sgd_workspace_bytes() >= 296 * 4
    # general attention: bad sizes / null pointers, and an empty batch is a no-op
    assert lib.ta3n_general_attn_fwd(None, 4, 0, 256, None, None, None, None, None, None, None, None) == 1
    assert lib.ta3n_general_attn_fwd(None, 4, 4, 256, None, None, None, None, None, None, None, None) == 1
    assert b"ta3n_general_attn_fwd" in lib.ta3n_last_error()
    assert lib.ta3n_general_attn_fwd(None, 0, 4, 256, None, None, None, None, None, None, None, None) == 0
    assert lib.ta3n_general_attn_bwd(None, 4, 4, 256, None, None, None, None, None, None, None, None, None, None, None,
                                     None, 0, None) == 1
    assert lib.ta3n_general_attn_bwd_workspace_bytes(256, 4, 256) >= 256 * 4 * 256 * 4
    assert lib.ta3n_relattn_bwd(None, 4, 4, 256, None, None, 3, None, None, None, None, None, None, 0.5, None, None,
                                None, None, None, None, 0, None) == 1
    # segment mean (avgpool): bad sizes / null pointers; an empty batch is a no-op
    assert lib.ta3n_segment_mean_fwd(None, 4, 0, 8, None, None) == 1
    assert lib.ta3n_segment_mean_fwd(None, 4, 5, 8, None, None) == 1
    assert lib.ta3n_segment_mean_bwd(None, 4, 5, 8, None, None) == 1
    assert lib.ta3n_segment_mean_fwd(None, 0, 5, 8, None, None) == 0
    # loss heads: a class count / batch of zero is rejected before anything is launched
    assert lib.ta3n_loss_fwd_bwd(None, None, None, None, None, 0, 0, 5, 4, 12, 0.003, 15, None, None, None, None,
                                 None, None, None, 0, None) == 1


def test_no_cpu_fallback_in_product_package():
    """The product package never imports the oracle and refuses CPU tensors."""
    import torch

    from ta3n_b200 import Ta3nError
    from ta3n_b200.models import VideoModel
    pkg = os.path.join(ROOT, "ta3n_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            assert "oracle" not in open(os.path.join(pkg, fn)).read().replace("the oracle", ""), fn
    m = VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    x = torch.zeros(2, 5, 2048)
    with pytest.raises(Ta3nError):
        m(x, x, [1, 1, 1], 0, True, False)     # model on CPU -> refuses


def test_unsupported_options_raise():
    from ta3n_b200.models import VideoModel
    for kw in (dict(frame_aggregation="rnn"), dict(frame_aggregation="avgpool", use_attn="general"), dict(use_bn="AdaBN"), dict(ens_DA="AutoDIAL"),
               dict(share_params="N"), dict(use_attn="general", use_attn_frame="TransAttn"), dict(baseline_type="tsn")):
        args = dict(num_class=5, baseline_type="video", frame_aggregation="trn-m", modality="RGB", verbose=False)
        args.update(kw)
        with pytest.raises(NotImplementedError):
            VideoModel(**args)
    with pytest.raises(ValueError):
        VideoModel(5, "video", "trn-m", "RGB", add_fc=0, verbose=False)


def test_avgpool_model_has_the_reference_parameters():
    """frame_aggregation='avgpool' (models.py:240-250, 285): shared_dim-wide video level, no TRN / relation layers."""
    from ta3n_b200.models import VideoModel
    from ta3n_b200.train import TrainStep
    m = VideoModel(5, "video", "avgpool", "RGB", train_segments=5, val_segments=5, fc_dim=128, verbose=False)
    sd = m.state_dict()
    assert not any(k.startswith(("TRN", "relation_domain_classifier_all", "bn_trn")) for k in sd)
    assert sd["fc_feature_domain_video.weight"].shape == (128, 128) and sd["fc_classifier_video_source.weight"].shape == (5, 128)
    assert len(m.path_parameters()) == 12
    with pytest.raises(NotImplementedError):
        TrainStep(m, 4, 4, beta=[0.75, 0.75, 0.5])


def test_general_attention_model_has_the_reference_parameters():
    """use_attn='general' (models.py:320-325): attn_layer = Linear(H,H), Tanh, Linear(H,1), appended to the operator's
    parameter list; TrainStep (the captured step of the shipped configuration) refuses the variant."""
    import torch

    from ta3n_b200.models import VideoModel
    from ta3n_b200.train import TrainStep
    m = VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, use_attn="general",
                   verbose=False)
    sd = m.state_dict()
    assert sd["attn_layer.0.weight"].shape == (256, 256) and sd["attn_layer.2.weight"].shape == (1, 256)
    assert sd["attn_layer.0.bias"].shape == (256,) and sd["attn_layer.2.bias"].shape == (1,)
    pp = m.path_parameters()
    assert len(pp) == 6 + 6 * 4 + 6 + 4 and pp[-4] is m.attn_layer[0].weight and pp[-1] is m.attn_layer[2].bias
    w = m.get_general_attn(torch.randn(3, 4, 256))
    assert w.shape == (3, 4, 1) and torch.allclose(w.sum(1), torch.ones(3, 1))
    with pytest.raises(NotImplementedError):
        TrainStep(m, 4, 4, beta=[0.75, 0.75, 0.5])


def test_relation_table_matches_survey_appendix_a():
    from ta3n_b200.functional import relation_set
    rs = relation_set(5)
    assert rs.tuples[1] == [(0, 1, 2, 3), (0, 1, 3, 4), (1, 2, 3, 4)]
    assert rs.tuples[3] == [(0, 1), (1, 2), (2, 3)]
    assert (rs.n_rel, rs.n_slots) == (10, 32)
    r9 = relation_set(9)
    assert (r9.n_rel, r9.n_slots) == (22, 114)


