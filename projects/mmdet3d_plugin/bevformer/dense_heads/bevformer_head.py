"""Drop-in module path for the detection head (the implementation lives in bevformer_b200/plugin/head.py)."""
from bevformer_b200.plugin.head import BEVFormerHead, BEVFormerHead_GroupDETR  # noqa: F401
