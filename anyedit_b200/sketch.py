"""AnyEdit's Canny sketch annotator on the H100 kernels: the condition image of the ``visual_sketch`` edits
(adaptive_editing_pipelines/visual_condition_tool.py:33-45 ``img2sketch``: cvtColor(BGR2GRAY), GaussianBlur((3, 3), 0),
Canny(50, 150), bitwise_not), equal to OpenCV's output on every pixel.

  ``detect(images)``                      uint8 BGR images [B, H, W, 3] (numpy, or a CUDA tensor) -> the uint8 sketches [B, H, W]
  ``img2sketch(image_path, output_path)`` the reference's function: reads with cv2, runs on the kernels, writes with cv2

Launch plan (DESIGN.md §10.7): one tile kernel from the BGR bytes to the per-pixel class (grey, blur, Sobel, non-maximum
suppression) and the union-find of each tile's candidates, then three launches of hysteresis on global labels.  CUDA only.
"""
import numbers

import numpy as np
import torch

from . import ops


def _check(images, low, high):
    if not (isinstance(images, (np.ndarray, torch.Tensor)) and images.dtype in (np.uint8, torch.uint8) and images.ndim == 4
            and images.shape[3] == 3):
        raise ValueError("sketch: expects uint8 BGR images [B, H, W, 3]")
    if not (isinstance(low, numbers.Integral) and isinstance(high, numbers.Integral) and 0 <= low <= high):
        raise ValueError(f"sketch: thresholds must be integers with 0 <= low <= high (got {low!r}, {high!r})")
    if not torch.cuda.is_available():
        raise RuntimeError("sketch runs on CUDA only (no CPU fallback)")


@torch.no_grad()
def detect(images, low=50, high=150):
    """255 - Canny(GaussianBlur(cvtColor(image, BGR2GRAY), (3, 3), 0), low, high) of each same-size uint8 BGR image
    [B, H, W, 3] (as ``cv2.imread`` gives it) -> uint8 [B, H, W]; numpy for numpy input, a CUDA tensor for a tensor."""
    _check(images, low, high)
    if isinstance(images, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(images)).cuda()
        return detect(x, low, high).cpu().numpy()
    if not images.is_cuda:
        raise RuntimeError("sketch runs on CUDA only (no CPU fallback); move the images to the GPU")
    images = images.contiguous()
    out = torch.empty(images.shape[:3], dtype=torch.uint8, device=images.device)
    ops.sketch(images, out, low, high)
    return out


def img2sketch(image_path, output_path):
    """visual_condition_tool.py img2sketch: the sketch of the image at ``image_path`` written to ``output_path``."""
    import cv2
    img = cv2.imread(image_path)
    cv2.imwrite(output_path, detect(img[None])[0])
