"""H100-native per-iteration hot path of crowsonkb/style-transfer-pytorch's StyleTransfer.stylize().

Import name: `style_transfer_b200` (see the loader module of that name at the repo root; this directory's
name is not a valid Python identifier)."""
from .style_transfer import STIterate, StyleTransfer, gen_scales, size_to_fit  # noqa: F401
