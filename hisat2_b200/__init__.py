"""hisat2_b200 -- H100-native (sm_90a) implementation of HISAT2's per-read alignment
hot path behind a C ABI (include/ht2gpu.h).  Python here is plumbing only:
ctypes bindings, batching helpers and the multi-GPU launcher glue."""
from .api import Index, ReadBatch, AlignResult, Ht2GpuError, load_library, format_align_summary, route_reads, READ_FILES, gunzip  # noqa: F401
