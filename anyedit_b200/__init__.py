"""anyedit_b200 -- H100-native AnySD denoising hot path (UNet forward + CFG/DDIM loop).

Public surface mirrors the reference's module API for this path:
    anyedit_b200.unet.UNetModel        <- ldm.modules.diffusionmodules.openaimodel.UNetModel
    anyedit_b200.ddim.DDIMSampler      <- ldm.models.diffusion.ddim.DDIMSampler
    anyedit_b200.diffusion.DiffusionWrapper / LatentDenoiser
                                       <- ldm.models.diffusion.ddpm.DiffusionWrapper / LatentDiffusion.apply_model
    anyedit_b200.anysd.MoE             <- AnySD.model.MoE (train.py:420-424, 694-695)
The same classes are importable under the reference's dotted paths prefixed with
``anyedit_b200.`` (e.g. ``anyedit_b200.ldm.modules.diffusionmodules.openaimodel.UNetModel``) so a
yaml ``target:`` only needs the prefix.
"""
__version__ = "0.1.0"
