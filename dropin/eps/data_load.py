"""eps.data_load -> the file helpers of aphantasia_b200.utils that cppn.py imports (cppn.py:29)."""
from aphantasia_b200.utils import basename, file_list, img_list, img_read, save_cfg  # noqa: F401
