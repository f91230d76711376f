"""pio-native-als: H100-native ALS hot path for PredictionIO's DASE engine templates.

The directory name follows the build contract (``incubator-predictionio_b200/``); because a
hyphen is not importable, the repo root carries ``pio_b200.py`` which loads this package under
the module name ``pio_b200``.

Layout:
  csrc/        CUDA kernels (sm_90a) + the C ABI (``include/pio_als.h``) -> libpio_als.so
  native.py    ctypes binding of the C ABI (stand-in for the JNI shim)
  synth.py     deterministic synthetic rating events (SURVEY 8(d))
  storage.py   Event / DataMap / BiMap / PEventStore mirror (host side of the ingest boundary)
  controller.py, workflow.py   DASE controller surface + CreateWorkflow/engine.json runner
  templates/   the recommendation / similarproduct / ecommerce / classification algorithms
"""
from . import native, synth  # noqa: F401

__all__ = ["native", "synth"]
