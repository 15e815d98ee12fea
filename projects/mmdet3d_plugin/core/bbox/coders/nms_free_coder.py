"""Drop-in module path for the NMS-free box coder (the implementation lives in bevformer_b200/plugin/head.py)."""
from bevformer_b200.plugin.head import NMSFreeCoder  # noqa: F401
