"""sparrowrecsys_b200 - H100-native CTR ranking forward path for SparrowRecSys.

Host side (this package): model specs, feature encoding, weight inventory, the
TF-free SavedModel reader, and the `tfrecmodel.*` call surface.  Device side
(`csrc/`): hand-written sm_90a kernels behind the C ABI in `include/srs_ctr.h`.
"""
from .spec import ModelSpec, baseline_spec, default_spec  # noqa: F401

__version__ = "0.1.0"
