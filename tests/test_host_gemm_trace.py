"""CPU: the GEMM phase timeline (tools/gemm_timeline.py) is compiled only into its own library, never into libb2d.so."""
import ctypes


def test_default_library_has_no_trace_code():
    from finetrainers_b200 import lib
    path = lib.build()
    assert not hasattr(ctypes.CDLL(path), "b2d_gemm_trace_set")
    with open(path, "rb") as fh:
        # the trace buffer's device symbol exists only in the -DB2D_GEMM_TRACE build
        assert b"g_gemm_trace" not in fh.read()
