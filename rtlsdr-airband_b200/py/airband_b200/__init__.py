"""airband_b200 — host-side Python mirror of the GPU demodulation path (tests and benchmarks drive the C ABI
through this; the product itself is the C-ABI shared library under rtlsdr-airband_b200/csrc)."""
from . import config, workloads  # noqa: F401
