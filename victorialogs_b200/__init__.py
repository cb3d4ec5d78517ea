"""victorialogs_b200: H100-native LogsQL block-scan / filter engine (drop-in for lib/logstorage's query hot path).

The package keeps its historical name.  The product is libvlscan.so (hand-written sm_90a CUDA kernels behind the C ABI of include/vlscan.h); `scan` is the
host-side mirror of the reference's filter / blockSearch interface on top of it."""
from . import scan  # noqa: F401
from .scan import Ctx, Filter, GenConfig, HostBlocks, Program, VlscanError, device_count, lib  # noqa: F401
