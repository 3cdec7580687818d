"""fp32 restatement of the reference's sampler (nerf/sd.py:176-199) as diffusers' DDIMScheduler runs it: set_timesteps for the three
timestep spacings, step() with eta = 0 and clip_sample off for epsilon and v_prediction, and the CFG loop on an oracle U-Net
(oracle/sd_ref.UNet2DConditionModel).  Written from diffusers' public scheduler source, independently of nerf/sd.py.  Test
infrastructure only."""
import math

import numpy as np
import torch

from oracle import sd_ref

T = 1000


def ddim_timesteps(n, spacing="leading", steps_offset=1):
    """DDIMScheduler.set_timesteps(n).timesteps"""
    if spacing == "leading":
        step_ratio = T // n
        ts = (np.arange(0, n) * step_ratio).round()[::-1].copy().astype(np.int64)
        ts += steps_offset
    elif spacing == "trailing":
        step_ratio = T / n
        ts = np.round(np.arange(T, 0, -step_ratio)).astype(np.int64)
        ts -= 1
    elif spacing == "linspace":
        ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
    else:
        raise ValueError(spacing)
    return ts


def ddim_step_ref(model_output, t, sample, n, prediction_type="epsilon", set_alpha_to_one=False, alphas=None):
    """DDIMScheduler.step(model_output, t, sample, eta=0) after set_timesteps(n), clip_sample and thresholding off"""
    alphas = sd_ref.alphas_cumprod() if alphas is None else alphas
    prev_t = t - T // n
    final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else alphas[0]
    alpha_prod_t = alphas[t]
    alpha_prod_t_prev = alphas[prev_t] if prev_t >= 0 else final_alpha_cumprod
    beta_prod_t = 1 - alpha_prod_t
    if prediction_type == "epsilon":
        pred_original_sample = (sample - beta_prod_t ** 0.5 * model_output) / alpha_prod_t ** 0.5
        pred_epsilon = model_output
    elif prediction_type == "v_prediction":
        pred_original_sample = alpha_prod_t ** 0.5 * sample - beta_prod_t ** 0.5 * model_output
        pred_epsilon = alpha_prod_t ** 0.5 * model_output + beta_prod_t ** 0.5 * sample
    else:
        raise ValueError(prediction_type)
    pred_sample_direction = (1 - alpha_prod_t_prev) ** 0.5 * pred_epsilon
    return alpha_prod_t_prev ** 0.5 * pred_original_sample + pred_sample_direction


def produce_latents_ref(unet, ctx, latents, num_inference_steps=50, guidance_scale=7.5, prediction_type="epsilon", spacing="leading",
                        steps_offset=1, set_alpha_to_one=False):
    """nerf/sd.py:176-199 for one prompt: ctx [2,77,D] (uncond, cond), latents [1,4,h,w]; fp32 throughout"""
    with torch.no_grad():
        for t in ddim_timesteps(num_inference_steps, spacing, steps_offset):
            t = int(t)
            noise_pred = unet(torch.cat([latents] * 2), torch.tensor([t], device=latents.device), ctx)
            noise_pred_uncond, noise_pred_text = noise_pred.chunk(2)
            noise_pred = noise_pred_text + guidance_scale * (noise_pred_text - noise_pred_uncond)
            latents = ddim_step_ref(noise_pred, t, latents, num_inference_steps, prediction_type, set_alpha_to_one)
    return latents


class UNet(sd_ref.UNet2DConditionModel):
    """the oracle U-Net with its time projection on t's device (no host round trip), so that the restatement can run on the GPU"""

    def time_proj(self, t):
        half = self.cfg["block_out"][0] // 2
        exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half
        emb = t.float()[:, None] * torch.exp(exponent)[None]
        return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)       # flip_sin_to_cos=True
