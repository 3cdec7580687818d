"""CPU checks of the sampler's host side: the DDIM schedule and update oracle (tests/sd_sample_ref.py), the schedule table nerf/sd.py
builds for mi3d_sd_sample against it, its C layout, the diffusers config mapping of from_pretrained with every refusal, the
safetensors reader, and the demo's argument parser."""
import ctypes
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sd_sample_ref as ref
from oracle import sd_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
Mi3dError = importlib.import_module("make-it-3d_b200._lib").Mi3dError


# ---- literal configs of the public checkpoints (unet/config.json, vae/config.json, scheduler/scheduler_config.json) ----
SD2_BASE_UNET = {"_class_name": "UNet2DConditionModel", "act_fn": "silu", "attention_head_dim": [5, 10, 20, 20],
                 "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False, "cross_attention_dim": 1024,
                 "down_block_types": ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"],
                 "downsample_padding": 1, "dual_cross_attention": False, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4,
                 "layers_per_block": 2, "mid_block_scale_factor": 1, "norm_eps": 1e-05, "norm_num_groups": 32, "out_channels": 4,
                 "sample_size": 64, "up_block_types": ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"],
                 "use_linear_projection": True}
SD21_UNET = dict(SD2_BASE_UNET, sample_size=96, upcast_attention=True)
SD15_UNET = {k: v for k, v in SD2_BASE_UNET.items() if k not in ("dual_cross_attention", "use_linear_projection")}
SD15_UNET.update(attention_head_dim=8, cross_attention_dim=768)
VAE = {"_class_name": "AutoencoderKL", "act_fn": "silu", "block_out_channels": [128, 256, 512, 512],
       "down_block_types": ["DownEncoderBlock2D"] * 4, "in_channels": 3, "latent_channels": 4, "layers_per_block": 2,
       "norm_num_groups": 32, "out_channels": 3, "sample_size": 512, "up_block_types": ["UpDecoderBlock2D"] * 4}
SD2_BASE_SCHED = {"_class_name": "PNDMScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear", "beta_start": 0.00085,
                  "clip_sample": False, "num_train_timesteps": 1000, "prediction_type": "epsilon", "set_alpha_to_one": False,
                  "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None}
SD21_SCHED = dict(SD2_BASE_SCHED, _class_name="DDIMScheduler", prediction_type="v_prediction")
SD15_SCHED = {k: v for k, v in SD2_BASE_SCHED.items() if k != "prediction_type"}


def test_timesteps_literal():
    lead = ref.ddim_timesteps(50, "leading", 1)
    assert lead[0] == 981 and lead[1] == 961 and lead[-1] == 1 and len(lead) == 50 and (np.diff(lead) == -20).all()
    trail = ref.ddim_timesteps(50, "trailing")
    assert trail[0] == 999 and trail[1] == 979 and trail[-1] == 19 and (np.diff(trail) == -20).all()
    lin = ref.ddim_timesteps(4, "linspace")
    assert lin.tolist() == [999, 666, 333, 0]
    assert ref.ddim_timesteps(3, "trailing").tolist() == [999, 666, 332]
    for n in (1, 3, 7, 50, 999):
        for sp, off in (("leading", 1), ("leading", 0), ("trailing", 0), ("linspace", 0)):
            assert sdm.ddim_timesteps(n, sp, off).tolist() == ref.ddim_timesteps(n, sp, off).tolist(), (n, sp, off)


def test_schedule_table_matches_the_oracle():
    a = sd_ref.alphas_cumprod()
    for n, sp, off, one in ((50, "leading", 1, False), (50, "trailing", 0, False), (7, "linspace", 0, True), (1, "leading", 1, False),
                            (1000, "leading", 0, False)):
        tab = sdm.ddim_schedule(n, sp, off, one)
        assert tab.dtype.itemsize == ctypes.sizeof(sdm.SDSchedule)
        ts = ref.ddim_timesteps(n, sp, off)
        assert tab["t"].tolist() == ts.tolist()
        assert np.array_equal(tab["alpha_t"], a[ts].numpy())
        for i, t in enumerate(ts):
            prev = t - 1000 // n
            want = float(a[prev]) if prev >= 0 else (1.0 if one else float(a[0]))
            assert tab["alpha_prev"][i] == np.float32(want), (n, sp, i)
    # the last leading step (t = 1, prev = -19) takes final_alpha_cumprod
    tab = sdm.ddim_schedule(50)
    assert tab["alpha_prev"][-1] == np.float32(a[0]) and sdm.ddim_schedule(50, set_alpha_to_one=True)["alpha_prev"][-1] == 1.0
    with pytest.raises(Mi3dError):
        sdm.ddim_schedule(1000, "leading", 1)          # t = 1000 is past the last train timestep
    for n in (0, 1001, 2.0):
        with pytest.raises(Mi3dError):
            sdm.ddim_timesteps(n)
    with pytest.raises(Mi3dError):
        sdm.ddim_timesteps(10, "karras")


def test_final_alpha_branch_of_the_step():
    g = torch.Generator().manual_seed(0)
    x, e = torch.randn(4, 8, generator=g), torch.randn(4, 8, generator=g)
    a = sd_ref.alphas_cumprod()
    got = ref.ddim_step_ref(e, 1, x, 50)                                    # prev = -19 -> alphas[0]
    x0 = (x - (1 - a[1]).sqrt() * e) / a[1].sqrt()
    assert torch.allclose(got, a[0].sqrt() * x0 + (1 - a[0]).sqrt() * e, rtol=0, atol=1e-6)
    assert torch.allclose(ref.ddim_step_ref(e, 1, x, 50, set_alpha_to_one=True), x0, rtol=0, atol=1e-6)
    # 1000 steps: prev = t - 1, the SDS path's denoise step (oracle/sd_ref.ddim_step_ref)
    for t in (0, 1, 399):
        assert torch.allclose(ref.ddim_step_ref(e, t, x, 1000), sd_ref.ddim_step_ref(e, t, x), rtol=0, atol=1e-6)


def test_v_prediction_algebra():
    """x_t = sqrt(a) x0 + sqrt(1-a) eps and v = sqrt(a) eps - sqrt(1-a) x0: the step's x0 / eps recovered from (x_t, v) are the true
    ones, so a step to alpha_prev = alpha_t reproduces x_t, and the step equals the epsilon step on the recovered eps"""
    g = torch.Generator().manual_seed(1)
    a = sd_ref.alphas_cumprod().double()
    for t in (1, 500, 999):
        x0, eps = torch.randn(4, 16, generator=g).double(), torch.randn(4, 16, generator=g).double()
        at = a[t]
        xt = at.sqrt() * x0 + (1 - at).sqrt() * eps
        v = at.sqrt() * eps - (1 - at).sqrt() * x0
        rec_x0 = at.sqrt() * xt - (1 - at).sqrt() * v
        rec_eps = at.sqrt() * v + (1 - at).sqrt() * xt
        assert torch.allclose(rec_x0, x0, atol=1e-10) and torch.allclose(rec_eps, eps, atol=1e-10)
        assert torch.allclose(at.sqrt() * rec_x0 + (1 - at).sqrt() * rec_eps, xt, atol=1e-10)
        n = 1000 // 20
        step_v = ref.ddim_step_ref(v, t, xt, n, "v_prediction", alphas=a)
        step_e = ref.ddim_step_ref(eps, t, xt, n, "epsilon", alphas=a)
        assert torch.allclose(step_v, step_e, atol=1e-10)


def test_config_mapping_of_the_public_checkpoints():
    assert sdm.unet_cfg_from_config(SD2_BASE_UNET) == sdm.sd20_unet_cfg()
    assert sdm.unet_cfg_from_config(SD21_UNET) == sdm.sd20_unet_cfg(96)
    assert sdm.unet_cfg_from_config(SD15_UNET) == sdm.sd15_unet_cfg()
    assert sdm.vae_cfg_from_config(VAE) == sdm.sd_vae_cfg()
    assert sdm.vae_cfg_from_config(dict(VAE, sample_size=768, scaling_factor=0.18215)) == sdm.sd_vae_cfg(768)
    assert sdm.scheduler_from_config(SD2_BASE_SCHED) == sdm.SD_SCHEDULER
    assert sdm.scheduler_from_config(SD15_SCHED) == sdm.SD_SCHEDULER
    assert sdm.scheduler_from_config(SD21_SCHED) == dict(sdm.SD_SCHEDULER, prediction_type="v_prediction")
    assert sdm.scheduler_from_config(dict(SD2_BASE_SCHED, timestep_spacing="trailing"))["timestep_spacing"] == "trailing"


@pytest.mark.parametrize("fn,cfg", [
    ("unet", dict(SD15_UNET, in_channels=9)),                                  # inpainting
    ("unet", dict(SD2_BASE_UNET, attention_head_dim=[5, 10, 20])),
    ("vae", dict(VAE, scaling_factor=0.13025)),
    ("sched", dict(SD2_BASE_SCHED, beta_schedule="linear")),
    ("sched", dict(SD2_BASE_SCHED, beta_end=0.02)),
    ("sched", dict(SD2_BASE_SCHED, num_train_timesteps=2000)),
    ("sched", dict(SD2_BASE_SCHED, trained_betas=[0.1] * 1000)),
    ("sched", dict(SD2_BASE_SCHED, clip_sample=True)),
    ("sched", {k: v for k, v in SD2_BASE_SCHED.items() if k != "clip_sample"}),   # DDIMScheduler's default clips
    ("sched", dict(SD2_BASE_SCHED, thresholding=True)),
    ("sched", dict(SD2_BASE_SCHED, prediction_type="sample")),
    ("sched", dict(SD2_BASE_SCHED, timestep_spacing="karras")),
])
def test_config_refusals(fn, cfg):
    f = dict(unet=sdm.unet_cfg_from_config, vae=sdm.vae_cfg_from_config, sched=sdm.scheduler_from_config)[fn]
    with pytest.raises(Mi3dError):
        f(cfg)


def test_safetensors_reader_and_bin_refusal(tmp_path):
    st = pytest.importorskip("safetensors.torch")
    g = torch.Generator().manual_seed(0)
    want = {"a.weight": torch.randn(3, 5, generator=g), "b.bias": torch.randn(7, generator=g).half(), "c": torch.arange(4)}
    (tmp_path / "unet").mkdir()
    st.save_file(want, str(tmp_path / "unet" / "diffusion_pytorch_model.fp16.safetensors"))
    got = sdm._read_weights(str(tmp_path / "unet"), "diffusion_pytorch_model")
    assert set(got) == set(want) and all(got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]) for k in want)
    (tmp_path / "vae").mkdir()
    (tmp_path / "vae" / "diffusion_pytorch_model.bin").write_bytes(b"\0")
    with pytest.raises(Mi3dError):
        sdm._read_weights(str(tmp_path / "vae"), "diffusion_pytorch_model")
    with pytest.raises(Mi3dError):
        sdm.StableDiffusion.from_pretrained(str(tmp_path / "missing"), "cpu")


def test_schedule_struct_layout(tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {',
           '  printf("%zu %zu %zu %zu\\n", sizeof(mi3d_sd_schedule), offsetof(mi3d_sd_schedule, t), offsetof(mi3d_sd_schedule, alpha_t),'
           ' offsetof(mi3d_sd_schedule, alpha_prev));', '  return 0;', '}']
    (tmp_path / "l.c").write_text("\n".join(src))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(tmp_path / "l.c"), "-o", str(tmp_path / "l")], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "l")], check=True, capture_output=True, text=True).stdout.split()]
    S = sdm.SDSchedule
    assert got == [ctypes.sizeof(S), S.t.offset, S.alpha_t.offset, S.alpha_prev.offset]
    assert sdm.ddim_schedule(3).dtype.itemsize == got[0]


def test_demo_help_parses():
    out = subprocess.run([sys.executable, "-m", "mi3d_b200.nerf.sd", "--help"], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    for flag in ("--ckpt", "--negative", "--workspace", "--sd_version", "-H", "-W", "--seeds", "--steps"):
        assert flag in out.stdout
