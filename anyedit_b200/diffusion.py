"""The ``apply_model`` boundary: conditioning mux + schedule buffers the samplers read.

Mirrors, without pytorch_lightning / omegaconf:
  * ``DiffusionWrapper.forward``          ldm/models/diffusion/ddpm.py:1324-1363 (conditioning keys)
  * ``LatentDiffusion.apply_model``       ddpm.py:854-869
  * ``DDPM.register_schedule``            ddpm.py:138-166 (float64 numpy -> fp32 buffers)
  * ``DDPM.q_sample``                     ddpm.py:356-359
VAE / text encoders (first_stage_model, cond_stage_model) are outside this path (SURVEY.md 8f);
``LatentDenoiser`` takes already-encoded conditioning, exactly what the samplers hand to apply_model.
"""
import importlib

import numpy as np
import torch
import torch.nn as nn

_KEYS = (None, "concat", "crossattn", "hybrid", "adm", "hybrid-adm", "crossattn-adm")


def instantiate_from_config(config):
    """ldm/util.py:74-89: {"target": "pkg.mod.Class", "params": {...}} -> object."""
    if "target" not in config:
        raise KeyError("Expected key `target` to instantiate.")
    module, cls = config["target"].rsplit(".", 1)
    return getattr(importlib.import_module(module), cls)(**config.get("params", dict()))


def make_beta_schedule(schedule, n_timestep, linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3):
    """ldm/modules/diffusionmodules/util.py:21-43 (float64)."""
    if schedule == "linear":
        betas = torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2
    elif schedule == "cosine":
        ts = torch.arange(n_timestep + 1, dtype=torch.float64) / n_timestep + cosine_s
        alphas = torch.cos(ts / (1 + cosine_s) * np.pi / 2).pow(2)
        alphas = alphas / alphas[0]
        betas = 1 - alphas[1:] / alphas[:-1]
        betas = np.clip(betas, a_min=0, a_max=0.999)
    elif schedule == "sqrt_linear":
        betas = torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64)
    elif schedule == "sqrt":
        betas = torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64) ** 0.5
    else:
        raise ValueError(f"schedule '{schedule}' unknown.")
    return betas.numpy()


class DiffusionWrapper(nn.Module):
    """ddpm.py:1324-1363.  ``diff_model_config`` may be a config dict or an already built module."""

    def __init__(self, diff_model_config, conditioning_key):
        super().__init__()
        if isinstance(diff_model_config, nn.Module):
            self.sequential_cross_attn = False
            self.diffusion_model = diff_model_config
        else:
            diff_model_config = dict(diff_model_config)
            self.sequential_cross_attn = diff_model_config.pop("sequential_crossattn", False)
            self.diffusion_model = instantiate_from_config(diff_model_config)
        self.conditioning_key = conditioning_key
        assert self.conditioning_key in _KEYS

    def forward(self, x, t, c_concat: list = None, c_crossattn: list = None, c_adm=None):
        key = self.conditioning_key
        if key is None:
            return self.diffusion_model(x, t)
        if key == "concat":
            return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t)
        if key == "crossattn":
            cc = torch.cat(c_crossattn, 1) if not self.sequential_cross_attn else c_crossattn
            return self.diffusion_model(x, t, context=cc)
        if key == "hybrid":
            return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t, context=torch.cat(c_crossattn, 1))
        if key == "hybrid-adm":
            assert c_adm is not None
            return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t, context=torch.cat(c_crossattn, 1), y=c_adm)
        if key == "crossattn-adm":
            assert c_adm is not None
            return self.diffusion_model(x, t, context=torch.cat(c_crossattn, 1), y=c_adm)
        if key == "adm":
            return self.diffusion_model(x, t, y=c_crossattn[0])
        raise NotImplementedError()


class LatentDenoiser(nn.Module):
    """The part of ``LatentDiffusion`` the samplers touch: schedule buffers, ``apply_model``, ``q_sample``.

    ``DDIMSampler(model)`` reads ``num_timesteps, betas, alphas_cumprod, alphas_cumprod_prev, device,
    parameterization, apply_model`` (+ ``q_sample`` for masked sampling) -- ddim.py:13-14, 27-34, 155, 188.
    """

    def __init__(self, unet_config, conditioning_key="hybrid", timesteps=1000, beta_schedule="linear",
                 linear_start=0.00085, linear_end=0.012, cosine_s=8e-3, parameterization="eps", given_betas=None,
                 first_stage_model=None, scale_factor=1.0):
        super().__init__()
        assert parameterization in ("eps", "x0", "v")
        self.parameterization = parameterization
        # optional first stage (anyedit_b200.autoencoder.AutoencoderKL) and the latent scale (0.18215 for SD, anydoor.yaml:17)
        self.first_stage_model, self.scale_factor = first_stage_model, float(scale_factor)
        self.model = DiffusionWrapper(unet_config, conditioning_key)
        self.conditioning_key = conditioning_key
        self.register_schedule(given_betas, beta_schedule, timesteps, linear_start, linear_end, cosine_s)

    @property
    def device(self):
        return self.betas.device

    @property
    def graph_safe(self):
        """True when the denoiser is an anyedit_b200 module: every op it issues is an async kernel
        launch on the current stream (no host syncs), so a sampler may capture it in a CUDA graph."""
        from .unet import UNetModel
        m = self.model.diffusion_model
        return isinstance(m, UNetModel) or getattr(m, "graph_safe", False)

    def graph_key(self):
        """Identity of the packed weights a captured CUDA graph would point at (parameter versions + device)."""
        m = self.model.diffusion_model
        return (tuple((str(p.device), p._version, p.data_ptr()) for p in m.parameters()).__hash__(), getattr(m, "_epoch", 0))

    def invalidate(self):
        m = self.model.diffusion_model
        if hasattr(m, "invalidate"):
            m.invalidate()

    def register_schedule(self, given_betas=None, beta_schedule="linear", timesteps=1000, linear_start=1e-4,
                          linear_end=2e-2, cosine_s=8e-3):
        betas = given_betas if given_betas is not None else make_beta_schedule(
            beta_schedule, timesteps, linear_start=linear_start, linear_end=linear_end, cosine_s=cosine_s)
        alphas = 1.0 - betas
        alphas_cumprod = np.cumprod(alphas, axis=0)
        alphas_cumprod_prev = np.append(1.0, alphas_cumprod[:-1])
        self.num_timesteps = int(betas.shape[0])
        self.linear_start, self.linear_end = linear_start, linear_end
        f32 = lambda a: torch.tensor(a, dtype=torch.float32)
        for name, val in (("betas", betas), ("alphas_cumprod", alphas_cumprod),
                          ("alphas_cumprod_prev", alphas_cumprod_prev),
                          ("sqrt_alphas_cumprod", np.sqrt(alphas_cumprod)),
                          ("sqrt_one_minus_alphas_cumprod", np.sqrt(1.0 - alphas_cumprod)),
                          ("log_one_minus_alphas_cumprod", np.log(1.0 - alphas_cumprod)),
                          ("sqrt_recip_alphas_cumprod", np.sqrt(1.0 / alphas_cumprod)),
                          ("sqrt_recipm1_alphas_cumprod", np.sqrt(1.0 / alphas_cumprod - 1))):
            if hasattr(self, name):
                setattr(self, name, f32(val).to(getattr(self, name).device))
            else:
                self.register_buffer(name, f32(val))

    def q_sample(self, x_start, t, noise=None):
        noise = torch.randn_like(x_start) if noise is None else noise
        shape = (t.shape[0],) + (1,) * (x_start.dim() - 1)
        return (self.sqrt_alphas_cumprod.gather(-1, t).reshape(shape) * x_start +
                self.sqrt_one_minus_alphas_cumprod.gather(-1, t).reshape(shape) * noise)

    def predict_eps_from_z_and_v(self, x_t, t, v):
        shape = (t.shape[0],) + (1,) * (x_t.dim() - 1)
        return (self.sqrt_alphas_cumprod.gather(-1, t).reshape(shape) * v +
                self.sqrt_one_minus_alphas_cumprod.gather(-1, t).reshape(shape) * x_t)

    def predict_start_from_z_and_v(self, x_t, t, v):
        shape = (t.shape[0],) + (1,) * (x_t.dim() - 1)
        return (self.sqrt_alphas_cumprod.gather(-1, t).reshape(shape) * x_t -
                self.sqrt_one_minus_alphas_cumprod.gather(-1, t).reshape(shape) * v)

    # ---- first stage (ddpm.py encode_first_stage / get_first_stage_encoding / decode_first_stage) ----
    def encode_first_stage(self, x):
        return self.first_stage_model.encode(x)

    def get_first_stage_encoding(self, encoder_posterior, noise=None):
        """scale_factor * posterior.sample() (a tensor is taken as the encoding itself), scaled inside the sampling kernel."""
        if isinstance(encoder_posterior, torch.Tensor):
            return self.scale_factor * encoder_posterior
        return encoder_posterior.sample(noise, scale=self.scale_factor)

    def decode_first_stage(self, z):
        """first_stage_model.decode(z / scale_factor); the factor rides in the 1x1 post_quant_conv weights."""
        return self.first_stage_model.decode(z, z_scale=1.0 / self.scale_factor)

    def apply_model(self, x_noisy, t, cond, return_ids=False):
        if not isinstance(cond, dict):
            if not isinstance(cond, list):
                cond = [cond]
            key = "c_concat" if self.model.conditioning_key == "concat" else "c_crossattn"
            cond = {key: cond}
        x_recon = self.model(x_noisy, t, **cond)
        if isinstance(x_recon, tuple) and not return_ids:
            return x_recon[0]
        return x_recon


class LatentInpaintDenoiser(LatentDenoiser):
    """ldm's ``LatentInpaintDiffusion`` (ddpm.py:1646-1690) on the sampler side: a ``hybrid`` denoiser whose UNet input is
    ``cat([x, mask, masked_image latents])`` in the order of ``concat_keys`` (the ``sd-v1-5-inpainting`` / ``sd-inpaint``
    layout: 9 UNet input channels).  The state dict is ldm's (``model.diffusion_model.*``, ``first_stage_model.*``), so the
    released checkpoint's ``state_dict`` loads with ``load_state_dict(..., strict=False)`` (the text encoder's keys are left
    over).  ``anyedit_b200.inpaint`` builds the concatenated channels."""

    # ldm yaml params (ddpm.py LatentDiffusion / LatentFinetuneDiffusion) that only concern training, logging or the stages
    # this class takes as modules: accepted and not used.  first_stage_config / cond_stage_config are not instantiated: pass
    # the built ``first_stage_model``; the text encoder stays outside the sampler path.
    _LDM_UNUSED = ("first_stage_config", "cond_stage_config", "first_stage_key", "cond_stage_key", "cond_stage_trainable",
                   "cond_stage_forward", "image_size", "channels", "monitor", "use_ema", "scale_by_std", "finetune_keys",
                   "keep_finetune_dims", "c_concat_log_start", "c_concat_log_end", "log_every_t", "scheduler_config",
                   "use_positional_encodings", "learn_logvar", "logvar_init", "loss_type", "load_only_unet", "ckpt_path",
                   "ignore_keys", "clip_denoised", "v_posterior", "l_simple_weight", "original_elbo_weight", "num_timesteps_cond")

    def __init__(self, unet_config, concat_keys=("mask", "masked_image"), masked_image_key="masked_image", conditioning_key="hybrid",
                 **kwargs):
        unknown = sorted(set(kwargs) - set(self._LDM_UNUSED) - {
            "timesteps", "beta_schedule", "linear_start", "linear_end", "cosine_s", "parameterization", "given_betas",
            "first_stage_model", "scale_factor"})
        if unknown:
            raise TypeError(f"LatentInpaintDiffusion: unexpected params {unknown}")
        kwargs = {k: v for k, v in kwargs.items() if k not in self._LDM_UNUSED}
        concat_keys = tuple(concat_keys)
        if masked_image_key not in concat_keys:
            raise ValueError(f"masked_image_key {masked_image_key!r} is not one of concat_keys {concat_keys}")
        if concat_keys != ("mask", "masked_image") or conditioning_key != "hybrid":
            raise NotImplementedError("LatentInpaintDiffusion: the mask + masked-image concatenation with hybrid conditioning "
                                      "(the SD inpainting checkpoints) is implemented")
        super().__init__(unet_config, conditioning_key=conditioning_key, **kwargs)
        self.concat_keys, self.masked_image_key = concat_keys, masked_image_key
