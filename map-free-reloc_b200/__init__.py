"""mfr_b200 — H100-native feature-matching + scale-from-depth relocalisation hot path.

Host side (Python, mirrors the reference's plugin surface) over hand-written sm_90a CUDA
behind the C ABI of ``libmfr_b200.so`` (``include/mfr_b200.h``). The directory is called
``map-free-reloc_b200``; import it as ``mfr_b200`` (see ``mfr_b200.py`` at the repo root).
"""
from . import lib  # noqa: F401
