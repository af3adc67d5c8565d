"""``from cgd.clip_util import MakeCutouts, encode_image_prompt, load_clip`` compatibility: the reference re-exports MakeCutouts there
(cgd/clip_util.py:13) and defines encode_image_prompt (cgd/clip_util.py:90-101; implemented in cgd.py / image_prompt.py) and load_clip
there (implemented in clip_model.py: a CLIP model whose encode_image runs this package's towers under torch.autograd).  CLIP weight
loading and the text tower live in ``cgd.py`` (`_load_clip_sd`, `_encode_text`): they run once per run, outside the hot path."""
from .guidance import MakeCutouts  # noqa: F401
from .cgd import encode_image_prompt  # noqa: F401,E402
from .clip_model import load_clip  # noqa: F401,E402
