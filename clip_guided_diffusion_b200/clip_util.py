"""``from cgd.clip_util import MakeCutouts, CLIP_NORMALIZE, encode_image_prompt, load_clip`` compatibility: the reference re-exports
MakeCutouts there (cgd/clip_util.py:13) and defines CLIP_NORMALIZE (cgd/clip_util.py:45), encode_image_prompt (cgd/clip_util.py:90-101;
implemented in cgd.py / image_prompt.py) and load_clip there (implemented in clip_model.py: a CLIP model whose encode_image runs this
package's towers under torch.autograd).  CLIP weight loading and the text tower live in ``cgd.py`` (`_load_clip_sd`, `_encode_text`): they
run once per run, outside the hot path."""
import torch as th

from .guidance import CLIP_MEAN, CLIP_STD, MakeCutouts  # noqa: F401
from .cgd import encode_image_prompt  # noqa: F401,E402
from .clip_model import load_clip  # noqa: F401,E402


class Normalize(th.nn.Module):
    """torchvision's ``Normalize(mean, std)`` on a tensor [..., C, H, W]: (x - mean[c]) / std[c], differentiable"""

    def __init__(self, mean, std):
        super().__init__()
        self.mean, self.std = list(mean), list(std)
        self._consts = {}

    def forward(self, tensor: th.Tensor) -> th.Tensor:
        key = (tensor.dtype, tensor.device)
        if key not in self._consts:
            self._consts[key] = tuple(th.as_tensor(v, dtype=tensor.dtype, device=tensor.device).view(-1, 1, 1) for v in (self.mean, self.std))
        mean, std = self._consts[key]
        return (tensor - mean) / std


CLIP_NORMALIZE = Normalize(CLIP_MEAN, CLIP_STD)
