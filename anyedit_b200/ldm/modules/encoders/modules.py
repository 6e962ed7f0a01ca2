"""Alias of ``ldm.modules.encoders.modules``: the condition encoders the ldm configs name as ``cond_stage_config`` targets
(AnyDoor's anydoor.yaml: ``FrozenDinoV2Encoder``)."""
from anyedit_b200.encoders import FrozenCLIPEmbedder, FrozenDinoV2Encoder  # noqa: F401
