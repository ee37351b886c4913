"""The int8-slice emulation is an argument of each fp64 call, not state of the calling thread: its size queries agree with
the rules they state (host only), and a call made on another host thread -- a fresh ``threading.Thread``, or autograd's
device thread running a backward -- gets the slice count it asks for."""
import threading

import pytest
import torch


def _oz_ws_bytes_1k(lib, rows, K, slices):
    return (lib.gpk_oz_ws_bytes(rows, K, slices) + 1023) // 1024 * 1024


def _gemm_need(lib, M, N, K, slices):
    """The emulated GEMM's rule: batch-1 products with M, N, K >= 256 and M N K >= 1.5e9, sliced in K chunks <= 65536."""
    if not 5 <= slices <= 8 or min(M, N, K) < 256 or M * N * K < 1.5e9:
        return 0
    passes = -(-K // 65536)
    kc = (K // passes + 127) // 128 * 128
    return _oz_ws_bytes_1k(lib, M, kc, slices) + lib.gpk_oz_ws_bytes(N, kc, slices)


def _trsm_need(lib, n, rows, slices):
    """The largest product of the recursive solve X L^T = B: the first h = (n / 128 // 2) 128 columns, the rows x (n - h) x h
    GEMM, then the last n - h columns."""
    if n <= 128:
        return 0
    h = n // 128 // 2 * 128
    return max(_gemm_need(lib, rows, n - h, h, slices), _trsm_need(lib, h, rows, slices),
               _trsm_need(lib, n - h, rows, slices))


def test_size_queries_follow_the_selection_rules():
    from stheno_b200 import _lib

    lib = _lib.load()
    for M, N, K in [(1152, 1024, 1280), (2048, 2048, 2048), (256, 384, 131200), (16384, 16384, 512), (1024, 1024, 1024),
                    (128, 8192, 8192), (8192, 8192, 128), (4096, 256, 1536)]:
        for slices in (0, 4, 5, 7, 8, 9):
            assert lib.gpk_gemm_nt_oz_ws_bytes(M, N, K, slices) == _gemm_need(lib, M, N, K, slices), (M, N, K, slices)
    assert lib.gpk_gemm_nt_oz_ws_bytes(1152, 1024, 1280, 8) > 0
    for n_pad in (128, 256, 384, 1920, 2048, 2176, 4096, 6016, 16384):
        for rows in (128, 256, 384, 2048, 4096):
            for slices in (0, 7, 8):
                assert lib.gpk_trsm_right_oz_ws_bytes(n_pad, rows, slices) == _trsm_need(lib, n_pad, rows, slices), (
                    n_pad, rows, slices)
    assert lib.gpk_trsm_right_oz_ws_bytes(2048, 2048, 7) > 0 and lib.gpk_trsm_right_oz_ws_bytes(4096, 128, 7) == 0
    # a factorisation: the slices of one 512-wide panel of all rows, from n_pad = 4096 those of a pair of panels
    for extra in (0, 128):
        for slices in (0, 7, 8):
            assert lib.gpk_potrf_oz_ws_bytes(1920, extra, slices) == 0
        assert lib.gpk_potrf_oz_ws_bytes(2048, extra, 0) == 0
        assert lib.gpk_potrf_oz_ws_bytes(2048, extra, 7) == lib.gpk_oz_ws_bytes(2048 + extra, 512, 7)
        R = 4096 + extra
        assert lib.gpk_potrf_oz_ws_bytes(4096, extra, 7) == _oz_ws_bytes_1k(lib, R, 1024, 7) + lib.gpk_oz_ws_bytes(R, 512, 7)


@pytest.mark.gpu
def test_every_host_thread_gets_the_emulation_it_asks_for():
    """An emulated ``gemm_nt`` (M N K >= 1.5e9) and a 2048-point ``logpdf`` backward, on the main thread and then on a fresh
    thread: the emulation kernel runs in both threads and during both backwards (autograd's device thread), and the two
    threads' products are bit-identical."""
    import stheno_b200 as S
    from stheno_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(0)
    A = torch.randn(1, 1152, 1280, device="cuda", dtype=torch.float64, generator=g)
    Bm = torch.randn(1, 1024, 1280, device="cuda", dtype=torch.float64, generator=g)
    x = torch.randn(2048, 4, device="cuda", dtype=torch.float64, generator=g)
    y = torch.randn(2048, device="cuda", dtype=torch.float64, generator=g)

    def emulated_launches(fn):
        ops.gemm_profile(True)
        try:
            out = fn()
            return out, ops.gemm_profile_read(1)[2]
        finally:
            ops.gemm_profile(False)

    def run(into):
        try:
            C, into["gemm"] = emulated_launches(lambda: ops.gemm_nt(A, Bm))
            into["C"] = C.clone()
            var = torch.tensor(1.3, device="cuda", dtype=torch.float64, requires_grad=True)
            lp = S.GP(var * S.EQ().stretch(2.0))(x, 0.1).logpdf(y)
            _, into["backward"] = emulated_launches(lp.backward)
        except BaseException as exc:  # reported by the main thread
            into["error"] = exc

    before = S.B.precision
    S.B.precision = "auto"
    try:
        main, other = {}, {}
        run(main)
        t = threading.Thread(target=run, args=(other,))
        t.start()
        t.join()
    finally:
        S.B.precision = before
    for res in (main, other):
        if "error" in res:
            raise res["error"]
    assert main["gemm"] > 0 and other["gemm"] > 0, (main["gemm"], other["gemm"])
    assert main["backward"] > 0 and other["backward"] > 0, (main["backward"], other["backward"])
    assert torch.equal(main["C"], other["C"])
