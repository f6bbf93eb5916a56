"""Host-side checks of image-to-video sampling: the timestep rule of the forward (one timestep per sample or per latent
frame), the conditioned step's C ABI entry point, and the input checks of ``generate_latents`` with a conditioning image
(CPU only)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tv(t, B=2, F=3, HW=4):
    from finetrainers_b200.model import timestep_values
    return timestep_values(t, B, F, HW)


def test_one_timestep_per_sample_in_any_shape():
    for t in (torch.tensor([437.25, 912.625]), torch.tensor([[437.25], [912.625]]), torch.tensor([400, 900])):
        got = _tv(t)
        assert got.dtype == torch.float32 and got.shape == (2,)
        assert torch.equal(got, t.reshape(2).float())


def test_per_token_timesteps_constant_per_sample_take_the_per_sample_plan():
    t = torch.tensor([437.25, 912.625]).view(2, 1, 1).expand(2, 12, 1)   # finetrainers' [B, S, 1]
    assert torch.equal(_tv(t), torch.tensor([437.25, 912.625]))
    long_t = (torch.tensor([0.4372, 0.9126]).view(2, 1, 1).expand(2, 12, 1) * 1000.0).long()
    assert torch.equal(_tv(long_t), torch.tensor([437.0, 912.0]))
    nan = torch.full((2, 12), float("nan"))                                # NaN codes compare equal bit for bit
    assert _tv(nan).shape == (2,)


def test_per_token_timesteps_that_differ_by_frame_give_one_per_frame():
    mask = torch.zeros(2, 3, 4)
    mask[:, 0] = 1.0                                                       # the conditioning frame
    t = torch.tensor(912.625) * (1 - mask.view(2, 12))                     # the image-to-video pipeline's [B, S]
    got = _tv(t)
    assert torch.equal(got, torch.tensor([0.0, 912.625, 912.625, 0.0, 912.625, 912.625]))
    frames = torch.tensor([[1.5, 2.5, 3.5], [4.0, 4.0, 5.0]]).repeat_interleave(4, 1)
    assert torch.equal(_tv(frames.unsqueeze(-1)), frames[:, ::4].reshape(6))
    # one sample varying is enough for the per-frame plan; the constant sample is repeated per frame
    mixed = torch.stack([torch.full((12,), 7.0), frames[1]])
    assert torch.equal(_tv(mixed), torch.tensor([7.0, 7.0, 7.0, 4.0, 4.0, 5.0]))


def test_signed_zeros_are_different_timesteps():
    t = torch.zeros(2, 12)
    t[1, 4:] = -0.0                                                        # sample 1, frames 1 and 2
    assert _tv(t).shape == (6,)


def test_timestep_varying_within_a_frame_names_sample_and_frame():
    t = torch.full((2, 12), 500.0)
    t[1, 9] = 499.0                                                        # sample 1, frame 2, token 1
    with pytest.raises(ValueError, match="frame 2 of sample 1"):
        _tv(t)
    t = torch.full((2, 12), 500.0)
    t[0, 5] = float("nan")
    with pytest.raises(ValueError, match="frame 1 of sample 0"):
        _tv(t)


@pytest.mark.parametrize("n", [1, 3, 6, 23, 25, 48])
def test_any_other_element_count_raises(n):
    with pytest.raises(ValueError, match="elements"):
        _tv(torch.zeros(n))


def test_conditioned_step_entry_point_is_declared_bound_and_wrapped():
    from finetrainers_b200 import lib, ops
    hdr = open(os.path.join(ROOT, "include", "b2d.h")).read()
    assert re.search(r"int b2d_cfg_euler_step_cond\(const void\* pred, float\* latents, void\* x_next, int32_t B, "
                     r"int64_t n, int64_t n_cond,\s*int32_t guided, float guidance, const float\* dt, void\* stream\);",
                     hdr)
    assert "Replaces:" in hdr.split("b2d_cfg_euler_step_cond(")[0].rsplit("/*", 1)[1]
    assert "b2d_cfg_euler_step_cond" in lib.EXPORTS
    assert callable(ops.cfg_euler_step_cond)
    src = open(os.path.join(ROOT, "finetrainers_b200", "csrc", "b2d_elem.cu")).read()
    assert "launch_k(cfg_euler_step_cond_kernel<true>" in src and "launch_k(cfg_euler_step_cond_kernel<false>" in src
    x = torch.zeros(2, 16)
    with pytest.raises(lib.B2DError):  # no CPU fallback
        ops.cfg_euler_step_cond(x.bfloat16(), x[:1], x.bfloat16(), 1, 16, 8, True, 3.0, torch.zeros(1))


class _NoLaunch(torch.nn.Module):
    """A transformer stand-in whose forward must never run: the checks come first."""

    def __init__(self):
        super().__init__()
        from finetrainers_b200.model import LTXConfig
        self.cfg = LTXConfig(in_channels=32)
        self.proj_in = torch.nn.Linear(1, 1)

    def forward(self, *a, **k):
        raise AssertionError("forward ran before the input checks")


def test_generate_latents_rejects_bad_image_input_before_launching():
    from finetrainers_b200.specification import LTXVideoModelSpecification
    spec = LTXVideoModelSpecification()
    tr = _NoLaunch()
    pe, pm = torch.zeros(1, 16, 4096), torch.ones(1, 16)
    ne, nm = torch.zeros(1, 16, 4096), torch.ones(1, 16)
    ok = dict(num_frames=9, height=64, width=96)                           # latent grid 2 x 2 x 3
    img, mean, std = torch.zeros(1, 32, 1, 2, 3), torch.zeros(32), torch.ones(32)

    def gen(**kw):
        args = dict(ok, image_latents=img, latents_mean=mean, latents_std=std)
        args.update(kw)
        spec.generate_latents(tr, pe, pm, ne, nm, **args)

    for bad in (torch.zeros(1, 32, 2, 2, 3), torch.zeros(1, 32, 2, 3), torch.zeros(2, 32, 1, 2, 3),
                torch.zeros(1, 16, 1, 2, 3), torch.zeros(1, 32, 1, 4, 3), torch.zeros(1, 32, 1, 2, 3, dtype=torch.int32)):
        with pytest.raises(ValueError, match="image_latents must be"):
            gen(image_latents=bad)
    with pytest.raises(ValueError, match="latents_mean"):
        gen(latents_mean=None)
    with pytest.raises(ValueError, match="latents_std"):
        gen(latents_std=None)
    with pytest.raises(ValueError, match="latents_mean must be"):
        gen(latents_mean=torch.zeros(31))
    with pytest.raises(ValueError, match="latents_std must be"):
        gen(latents_std=torch.ones(1, 32))
    with pytest.raises(ValueError, match="latents_std must be"):
        gen(latents_std=torch.ones(32, dtype=torch.int64))
    with pytest.raises(ValueError, match="num_frames >= 9"):
        gen(num_frames=1)
    with pytest.raises(ValueError, match="latents must be packed"):
        gen(latents=torch.zeros(1, 5, 32))
    with pytest.raises(ValueError, match="which was not given"):
        spec.generate_latents(tr, pe, pm, ne, nm, latents_mean=mean, latents_std=std, **ok)
    # a good call passes every check and reaches the transformer (the stand-in then refuses to run)
    with pytest.raises(AssertionError, match="forward ran"):
        gen(latents_mean=[0.0] * 32)
