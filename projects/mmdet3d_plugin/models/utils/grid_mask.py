"""Drop-in module path for GridMask (the implementation lives in bevformer_b200/plugin/grid_mask.py).  The reference's
per-image ``Grid`` class, which no pipeline uses, is not re-exported."""
from bevformer_b200.plugin.grid_mask import GridMask  # noqa: F401
