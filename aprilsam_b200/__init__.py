"""aprilsam_b200: H100-native (sm_90a) replacement for AprilSAM's april_graph_cholesky{,_inc} path.

The product is the C/CUDA shared library `libaprilsam_b200.so` (drop-in for the reference's
libaprilsam public API, see include/aprilsam/aprilsam.h and INTEGRATION.md).  This Python
package only holds build tooling, the ctypes mirror of the C API used by tests/bench, and
the synthetic-data generators.
"""
__all__ = ["harness", "datasets", "build"]
