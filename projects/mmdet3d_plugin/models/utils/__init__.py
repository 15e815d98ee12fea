# Same import path as the reference package for GridMask only (run_time, RelPositionEmbedding and save_tensor stay the
# reference's own).
from .grid_mask import GridMask
