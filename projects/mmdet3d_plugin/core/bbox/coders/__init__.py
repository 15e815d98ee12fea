# Same import surface as the reference package of this path (the implementation lives in bevformer_b200/plugin/head.py).
from .nms_free_coder import NMSFreeCoder
