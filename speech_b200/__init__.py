"""speech_b200 - H100-native (sm_90a) replacement for the data-parallel hot path of awni/speech.

Layout (SURVEY.md §8):
    csrc/        hand-written CUDA kernels + the C ABI (include/speech_b200.h), built in-tree
    _lib.py      ctypes binding of that ABI (no CPU fallback)
    functions/   operator-level drop-ins: functions.ctc.CTCLoss, transducer.* (reference imports)
    models/      host-side mirror of speech.models.{Model,CTC,Seq2Seq,Transducer}
    loader.py    input pipeline (BatchPrefetcher); features.py  GPU featuriser (log_specgram)
    utils/       save / load / compute_cer, as `speech/__init__.py` re-exports them
"""
__version__ = "0.1.0"

from .utils.io import load, save                 # noqa: E402,F401  (speech/__init__.py:1)
from .utils.score import compute_cer             # noqa: E402,F401  (speech/__init__.py:2)
