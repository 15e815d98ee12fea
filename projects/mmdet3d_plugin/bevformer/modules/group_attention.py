"""Drop-in module path: the implementation lives in bevformer_b200/plugin/decoder.py."""
from bevformer_b200.plugin.decoder import GroupMultiheadAttention  # noqa: F401
