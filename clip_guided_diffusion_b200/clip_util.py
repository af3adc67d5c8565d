"""``from cgd.clip_util import MakeCutouts, encode_image_prompt`` compatibility: the reference re-exports MakeCutouts there
(cgd/clip_util.py:13) and defines encode_image_prompt there (cgd/clip_util.py:90-101; implemented in cgd.py / image_prompt.py).  CLIP weight loading
and the text tower live in ``cgd.py`` (`_load_clip_sd`, `_encode_text`): they run once per run, outside the hot path."""
from .guidance import MakeCutouts  # noqa: F401
from .cgd import encode_image_prompt  # noqa: F401,E402
