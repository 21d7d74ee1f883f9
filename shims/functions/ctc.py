"""Import-compatible stand-in for warp-ctc's pytorch_binding module `functions.ctc`, which the
reference imports at speech/models/ctc_model.py:9.  Re-exports the sm_90a implementation."""
from speech_b200.functions.ctc import CTCLoss  # noqa: F401
