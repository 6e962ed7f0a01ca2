"""Alias of the sampler-facing part of ``ldm.models.diffusion.ddpm``."""
from anyedit_b200.diffusion import DiffusionWrapper, LatentDenoiser, LatentInpaintDenoiser  # noqa: F401

LatentDiffusion = LatentDenoiser
LatentInpaintDiffusion = LatentInpaintDenoiser
