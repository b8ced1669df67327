"""caffeonspark_b200 -- H100-native gradient synchronisation for CaffeOnSpark.

Host-side mirror (Python, for tests and the benchmark harness) of the
reference's ``com.yahoo.ml.jcaffe.CaffeNet`` JNI class over the C ABI of
``libcaffedistri_b200.so`` (see include/caffedistri_b200.h).  All compute is
in the CUDA library; there is no CPU fallback anywhere in this package.
"""
from .caffenet import (CaffeNet, CosError, PeerAdapter, SolverDesc, chunk, learning_rate, parse_solver,  # noqa: F401
                       input_transform_plan, native_producer_plan, read_caffemodel_blob, read_solverstate)
from ._lib import build_library, library_path  # noqa: F401

__all__ = ["CaffeNet", "CosError", "PeerAdapter", "SolverDesc", "chunk", "learning_rate", "parse_solver",
           "input_transform_plan", "native_producer_plan", "read_caffemodel_blob", "read_solverstate",
           "build_library", "library_path"]
