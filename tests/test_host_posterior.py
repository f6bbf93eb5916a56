"""CPU: training from precomputed VAE moments (``compute_posterior=False``) - the test-side posterior sample against the
reference's own ``DiagonalGaussianDistribution`` (tests/golden/posterior_golden.pt, made by make_posterior_golden.py),
moments items through the precomputed feed unchanged, and the moments shape checks of the specification and the step."""
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = dict(in_channels=8, out_channels=8, num_attention_heads=2, attention_head_dim=64, cross_attention_dim=128,
             num_layers=1, caption_channels=32)


@pytest.fixture(scope="module")
def posterior_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "posterior_golden.pt"), weights_only=False)["cases"]


def _bits_equal(a, b):
    """Bit-identical bf16 tensors, except that any NaN matches any NaN (NaN in, NaN out)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.view(torch.int16)[~na], b.view(torch.int16)[~nb])


def test_golden_covers_the_clamp_edges(posterior_golden):
    assert len(posterior_golden) >= 3
    assert any(c["shape"][1] == 128 for c in posterior_golden)
    assert any((c["shape"][2] * c["shape"][3] * c["shape"][4]) % 2 for c in posterior_golden)
    for c in posterior_golden:
        lv = c["moments"][:, c["shape"][1]:].float()
        assert (lv < -30).any() and (lv > 20).any() and (lv == float("inf")).any() and (lv == float("-inf")).any()
        assert torch.isnan(lv).any() and torch.isnan(c["sample"]).any()


def test_posterior_restatement_is_bit_identical_to_the_reference(posterior_golden):
    from _posterior import posterior_sample
    for c in posterior_golden:
        assert c["moments"].dtype == torch.bfloat16 and c["sample"].dtype == torch.bfloat16
        got = posterior_sample(c["moments"], generator=torch.Generator().manual_seed(c["seed"]))
        assert _bits_equal(got, c["sample"]), c["shape"]
        assert _bits_equal(posterior_sample(c["moments"], eps=c["eps"]), c["sample"]), c["shape"]
        # the draw is torch.randn on the moments' dtype: the same stream as normal_() on a bf16 buffer (the step's draw)
        eps = torch.empty(c["eps"].shape, dtype=torch.bfloat16).normal_(generator=torch.Generator().manual_seed(c["seed"]))
        assert torch.equal(eps.view(torch.int16), c["eps"].view(torch.int16))


def test_moments_items_pass_the_precomputed_feed_unchanged(tmp_path):
    """Moments items in the reference's precomputation layout ({data_type}-{index}.pt dicts) through both readers, the
    resolution sampler bucketing on dims 2, 3, 4 of the leader and collate: the moments reach the step bit for bit, with
    their 2C channels."""
    from finetrainers_b200.data import PrecomputedOnceReader, PrecomputedReader, ResolutionSampler, collate, save_item
    g = torch.Generator().manual_seed(0)
    shapes = [(3, 4, 6), (2, 4, 6), (3, 4, 6), (2, 4, 6)]
    items = []
    for i, (F, H, W) in enumerate(shapes):
        it = {"latents": torch.randn(1, 16, F, H, W, generator=g).bfloat16(), "num_frames": F, "height": H, "width": W,
              "latents_mean": torch.randn(1, 8, generator=g), "latents_std": torch.rand(1, 8, generator=g) + 0.5}
        save_item(it, i, tmp_path, "latent")
        items.append(it)
    for reader in (PrecomputedReader(tmp_path, "latent"), PrecomputedOnceReader(tmp_path, "latent")):
        sampler = ResolutionSampler(batch_size=2, dim_keys={"latents": (2, 3, 4)})
        batches = []
        it = iter(reader)
        for _ in range(len(shapes)):
            sampler.consume(next(it))
            while sampler.is_ready:
                batches.append(collate(list(sampler.get_batch()[0])))
        assert len(batches) == 2
        for b, idx in zip(batches, ([0, 2], [1, 3])):
            want = torch.cat([items[i]["latents"] for i in idx])
            assert b["latents"].shape == (2, 16) + shapes[idx[0]]
            assert torch.equal(b["latents"].view(torch.int16), want.view(torch.int16))
            assert torch.equal(b["latents_mean"], items[idx[0]]["latents_mean"])   # taken from the first item
            assert b["num_frames"] == shapes[idx[0]][0]


class _Cfg:
    in_channels = 8


class _NoTransformer:
    """A transformer stand-in that fails the test if the specification gets as far as calling it."""
    cfg = _Cfg()

    def __call__(self, *a, **k):
        raise AssertionError("the transformer ran before the moments shape was checked")


@pytest.mark.parametrize("channels", [15, 8, 32, 18])
def test_specification_refuses_bad_moment_channels(channels):
    from finetrainers_b200.specification import LTXVideoModelSpecification
    spec = LTXVideoModelSpecification()
    lat = {"latents": torch.zeros(1, channels, 2, 2, 2), "latents_mean": torch.zeros(1, 8), "latents_std": torch.ones(1, 8)}
    with pytest.raises(ValueError, match=rf"\(1, {channels}, 2, 2, 2\)"):
        spec.forward(_NoTransformer(), {}, lat, torch.zeros(1), compute_posterior=False)


def _cpu_step():
    from finetrainers_b200.model import B200LTXTransformer, LTXConfig
    from finetrainers_b200.trainer import SFTTrainStep
    bm = B200LTXTransformer(LTXConfig(**SMALL), torch.bfloat16, "cpu")
    bm.add_adapter(16, 16)
    bm.prepare()
    return SFTTrainStep(bm, flow_weighting_scheme="none")


@pytest.mark.parametrize("channels", [15, 8, 32])
def test_train_step_refuses_bad_moment_channels_before_any_launch(channels):
    st = _cpu_step()
    cond = {"encoder_hidden_states": torch.zeros(1, 4, 32, dtype=torch.bfloat16)}
    lat = {"latents": torch.zeros(1, channels, 2, 2, 2, dtype=torch.bfloat16)}
    with pytest.raises(ValueError, match=rf"\(1, {channels}, 2, 2, 2\)"):
        st.train_step(cond, lat, compute_posterior=False)
    assert not st._static and st.micro == 0


def test_moments_and_latents_inputs_never_share_buffers():
    """A moments input [B, 2C, ...] and a latents input of the same latent shape get their own static buffers (and so
    their own CUDA graphs): the graph key carries the input kind."""
    st = _cpu_step()
    k_lat, b_lat = st._buffers(1, 8, 2, 2, 2, 4, 32)
    k_mom, b_mom = st._buffers(1, 8, 2, 2, 2, 4, 32, True)
    assert k_lat != k_mom and len(st._static) == 2
    assert "latents" in b_lat and "moments" not in b_lat
    assert b_mom["moments"].shape == (1, 16, 2, 2, 2) and b_mom["eps"].shape == (1, 8, 2, 2, 2) and "latents" not in b_mom
