"""The DPT-Hybrid oracle (oracle/dpt_ref.py) against an independent implementation: transformers' `DPTForDepthEstimation` at the
hybrid (BiT-backbone) configuration of DPT-Hybrid, on the CPU with transformers' own seeded initialisation."""
import pytest
import torch

from oracle import dpt_ref

transformers = pytest.importorskip("transformers")


def _hf_config():
    return transformers.DPTConfig(
        is_hybrid=True,
        backbone_config=transformers.BitConfig(global_padding="same", layer_type="bottleneck", depths=[3, 4, 9],
                                               out_features=["stage1", "stage2", "stage3"], embedding_dynamic_padding=True),
        backbone_featmap_shape=[1, 1024, 24, 24], neck_hidden_sizes=[256, 512, 768, 768], reassemble_factors=[1, 1, 1, 0.5],
        readout_type="project", backbone_out_indices=[2, 5, 8, 11], neck_ignore_stages=[0, 1], fusion_hidden_size=256, image_size=384,
        layer_norm_eps=1e-6)


@pytest.fixture(scope="module")
def hf():
    torch.manual_seed(0)
    return transformers.DPTForDepthEstimation(_hf_config()).eval()


def test_name_map_is_one_to_one(hf):
    sd = hf.state_dict()
    assert len(sd) == 414 and sum(v.numel() for v in sd.values()) == 122_377_985
    m = dpt_ref.hf_name_map()
    targets = [n for v in m.values() for n in (v if isinstance(v, tuple) else (v,))]
    assert sorted(targets) == sorted(sd)
    ref = dict(dpt_ref.param_shapes(), **dpt_ref.ignored_shapes())
    assert set(m) == {n for n in ref if not n.startswith("pretrained.model.head.")}
    conv = dpt_ref.from_hf_state_dict(sd)
    for n, t in conv.items():
        assert tuple(t.shape) == tuple(ref[n]), n
    # the forward reads every tensor but the ignored ones
    assert set(dpt_ref.param_shapes()) == {n for n in conv if not n.startswith(dpt_ref.IGNORED_PREFIXES)}


def test_forward_matches_transformers(hf):
    # in float64: fp32 rounding alone moves either implementation by ~2.4e-5 relative L2 on this 100-layer network, which would hide
    # a structural difference of that size; in float64 the two agree to ~3e-14
    torch.set_num_threads(min(32, torch.get_num_threads()))
    x = torch.randn(1, 3, 384, 384, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    p = {k: v.double() for k, v in dpt_ref.from_hf_state_dict(hf.state_dict()).items()}
    with torch.no_grad():
        want = hf.double()(pixel_values=x).predicted_depth
        got = dpt_ref.forward(p, x)
    hf.float()
    err = float((got - want).norm() / want.norm())
    print(f"oracle vs transformers rel-L2 {err:.2e} (float64), positive pixels {float((want > 0).double().mean()):.3f}")
    assert got.shape == want.shape == (1, 384, 384)
    assert err < 1e-9


def test_default_init_is_not_degenerate():
    torch.set_num_threads(min(32, torch.get_num_threads()))
    x = torch.randn(1, 3, 384, 384, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        out = dpt_ref.forward(dpt_ref.default_init(0), x)
    frac = float((out > 0).double().mean())
    print(f"positive pixels under the seeded stand-in weights: {frac:.3f}")
    assert 0.2 < frac and float(out.std()) > 0
