"""CPU tests of the linear SVM at ILSVRC and iNaturalist scale: the workspace of the GEMM row blocks and of the class
blocks against svm_scale_oracle, the widest fixed-order class block, the block-size rule of linear_svm_fit, and the
argument checks of se_linear_svm_fit_classes."""
import os

import pytest

import svm_oracle
import svm_scale_oracle as sso

# (N, D, C) of the feature sets the SVM path is used on: ILSVRC and iNaturalist 2018 / 2019 at ResNet-50's avg_pool
# width and at the embedding widths, and an ILSVRC problem with --augmentation_epochs 2
TABLE = [(1281167, 2048, 1000), (437513, 2048, 8142), (437513, 1024, 8142), (1281167, 1000, 1000), (265213, 2048, 1010),
         (2 * 1281167, 1000, 1000)]


def _lib():
    from semantic_embeddings_b200 import _lib as L
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    L.load()
    return L


@pytest.mark.parametrize('N,D,C', TABLE + [(1100000, 2048, 64), (270000, 256, 8142), (20000, 640, 16), (20000, 640, 33),
                                           (2 ** 20, 2048, 16), (2 ** 20 + 1, 2048, 16), (2 ** 20 - 32, 2048, 17)])
def test_workspace_matches_the_extended_layout(N, D, C):
    """se_linear_svm_workspace_bytes and se_linear_svm_classes_workspace_bytes end where the extended layout says, with
    every GEMM call below 2^31 elements of X, S and R and Np the row blocks' sum; below 2^31 elements the layout is
    svm_oracle's."""
    lib = _lib().load()
    dims, regions, total = sso.svm_layout(N, D, C)
    assert int(lib.se_linear_svm_workspace_bytes(N, D, C)) == total
    assert int(lib.se_linear_svm_classes_workspace_bytes(N, D, C)) == total
    assert all(off % 256 == 0 for _, off, _, _ in regions)
    rb, nblk, Np = dims['rb'], dims['nblk'], dims['Np']
    assert rb * nblk == Np >= max(N, 32) and rb >= 32
    assert rb * max(dims['Dp'], dims['Cp']) < 2 ** 31
    if max(N, 32) * max(dims['Dp'], dims['Cp']) < 2 ** 31:
        assert nblk == 1 and svm_oracle.svm_layout(N, D, C)[2] == total
    else:
        assert nblk >= 2 and rb % 64 == 0 and Np - max(N, 32) < 64 * nblk


def test_row_block_edges():
    """The first N whose rows x Dp reaches 2^31 takes two blocks; one row fewer keeps one block and its layout."""
    edge = 2 ** 31 // 2048
    assert sso.row_blocks(edge - 1, 2048, 16) == (edge - 1, edge - 1, 1)
    Np, rb, nblk = sso.row_blocks(edge, 2048, 16)
    assert nblk == 2 and rb * 2048 < 2 ** 31 <= edge * 2048
    Np, rb, nblk = sso.row_blocks(270000, 256, 8142)          # Cp = 8144 decides
    assert (Np, rb, nblk) == (270080, 135040, 2)


def test_widest_fixed_order_class_block():
    """se_linear_svm_block_classes: the whole problem where (D+1) x C fits the fixed-order workspace (two slices of
    Dp Cp + Cp floats in 8 M), else the widest multiple of 16 that does; the boundary matches
    test_svm_fixed_order_refusal_boundary's (Dp, Cp) = (4092, 1024)."""
    lib = _lib().load()
    ws = 8 << 20
    fits = lambda Dp, Cp: 2 * (Dp * Cp + Cp) <= ws
    assert lib.se_linear_svm_block_classes(64, 4092, 1024) == 1024
    assert lib.se_linear_svm_block_classes(64, 4096, 1024) == 1008
    for N, D, C in TABLE + [(50000, 640, 100), (20000, 2048, 555)]:
        cb = int(lib.se_linear_svm_block_classes(N, D, C))
        Dp = (D + 3) // 4 * 4
        if fits(Dp, (C + 15) // 16 * 16):
            assert cb == C, (N, D, C)
        else:
            assert cb % 16 == 0 and fits(Dp, cb) and not fits(Dp, cb + 16), (N, D, C, cb)
    assert lib.se_linear_svm_block_classes(437513, 2048, 8142) == 2032
    assert lib.se_linear_svm_block_classes(0, 2048, 10) == 0


def test_block_size_rule():
    from semantic_embeddings_b200.classification import svm_block_classes
    ws = lambda c: 1000 + 10 * ((c + 15) // 16 * 16)
    assert svm_block_classes(100, 100, ws, 10 ** 9) == 100
    assert svm_block_classes(100, 100, ws, 10 ** 9, max_block_classes=33) == 33
    assert svm_block_classes(100, 100, ws, 10 ** 9, max_block_classes=16) == 16
    assert svm_block_classes(100, 100, ws, 10 ** 9, max_block_classes=500) == 100
    assert svm_block_classes(8142, 2032, ws, 10 ** 9) == 2032                  # the fixed-order limit
    assert svm_block_classes(8142, 2032, ws, 1000 + 10 * 512) == 512           # free memory
    assert svm_block_classes(100, 100, ws, 1000 + 10 * 40) == 32               # memory below C: a multiple of 16
    assert svm_block_classes(100, 100, ws, 1000) == 0                          # nothing fits
    assert svm_block_classes(100, 100, lambda c: 0, 10 ** 9) == 0              # no workspace exists


def test_block_size_rule_at_ilsvrc_and_inaturalist_scale():
    """With the library's workspace sizes: ILSVRC's whole problem needs 26.2 GB besides X (10.5 GB of it the packed X)
    and fits one block in 60 GB; iNaturalist 2018 takes blocks of the fixed-order width, or narrower ones when memory is
    short."""
    from semantic_embeddings_b200.classification import svm_block_classes
    lib = _lib().load()
    gb = 10 ** 9
    for (N, D, C), one in (((1281167, 2048, 1000), True), ((437513, 2048, 8142), False)):
        ws = lambda c: int(lib.se_linear_svm_classes_workspace_bytes(N, D, c))
        fixed = int(lib.se_linear_svm_block_classes(N, D, C))
        cb = svm_block_classes(C, fixed, ws, 60 * gb)
        assert (cb == C) == one and cb > 0 and ws(cb) <= 60 * gb
        small = svm_block_classes(C, fixed, ws, ws(16) + 1)
        assert small == 16
    assert abs(lib.se_linear_svm_workspace_bytes(1281167, 2048, 1000) - 26.2 * gb) < 0.05 * gb
    assert abs(lib.se_linear_svm_workspace_bytes(437513, 2048, 8142) - 47.3 * gb) < 0.05 * gb


def _fit_classes(L, x, ldx, N, D, labels, C, c0, cb, packed=0, ws=256):
    return L.load().se_linear_svm_fit_classes(x, ldx, N, D, labels, C, c0, cb, 1.0, 1e-4, 10, 256, 256, None, None, ws,
                                              packed, None)


def test_fit_classes_argument_checks():
    """c0 outside [0, C), cb outside (0, C], missing pointers and a misaligned workspace are refused before any device work."""
    L = _lib()
    msg = lambda: L.load().se_last_error().decode()
    for c0, cb in ((-1, 16), (100, 16), (101, 16), (0, 0), (5, -3), (0, 101), (50, 2 ** 31 - 1)):
        assert _fit_classes(L, 256, 64, 1000, 64, 256, 100, c0, cb) == -1, (c0, cb)
        assert 'c0' in msg() and 'cb' in msg()
    assert _fit_classes(L, 256, 64, 1000, 64, None, 100, 0, 16) == -1 and 'null' in msg()     # labels
    assert _fit_classes(L, None, 64, 1000, 64, 256, 100, 0, 16) == -1 and 'null' in msg()     # X, not packed
    assert _fit_classes(L, 256, 63, 1000, 64, 256, 100, 0, 16) == -1 and 'ldx' in msg()
    assert _fit_classes(L, 256, 64, 1000, 64, 256, 100, 0, 16, ws=512 + 8) == -1 and 'aligned' in msg()
    assert _fit_classes(L, 256, 64, 1000, 64, 256, 0, 0, 16) == -1


@pytest.mark.parametrize('N,D,C', TABLE)
def test_table_shapes_pass_the_argument_checks(N, D, C):
    """The ILSVRC / iNaturalist shapes that se_linear_svm_fit refused with 'N x D and N x C must stay below 2^31' pass
    every shape rule now, read through the host-only queries: the layout exists (what the fit's last argument check
    requires) and some class block fits the fixed-order workspace.  The fit itself is not called here: past its argument
    checks it works on device memory."""
    lib = _lib().load()
    assert int(lib.se_linear_svm_workspace_bytes(N, D, C)) == sso.svm_layout(N, D, C)[2] > 0
    cb = int(lib.se_linear_svm_block_classes(N, D, C))
    assert 0 < cb <= C
    assert int(lib.se_linear_svm_classes_workspace_bytes(N, D, cb)) == sso.svm_layout(N, D, cb)[2]


def test_what_the_layout_cannot_hold_is_refused_before_any_device_work():
    """Rows that padded to whole GEMM row blocks pass 2^31, and block widths whose padding overflows an int, have no
    workspace (0 bytes) and are refused by the argument checks, which run before any device call."""
    L = _lib()
    lib = L.load()
    N = 2 ** 31 - 1
    assert lib.se_linear_svm_workspace_bytes(N, 2048, 1000) == 0
    assert lib.se_linear_svm_fit(256, 2048, N, 2048, 256, 1000, 1.0, 1e-4, 10, 256, None, None, None, 256, None) == -1
    assert 'row blocks' in lib.se_last_error().decode()
    assert lib.se_linear_svm_classes_workspace_bytes(1000, 64, 2 ** 31 - 1) == 0
    assert lib.se_linear_svm_block_classes(1000, 2 ** 31 - 1, 100) == 0


def test_raw_fit_still_refuses_the_fixed_order_boundary():
    """se_linear_svm_fit keeps its refusal of (Dp, Cp) = (4096, 1024) with SE_ERR_UNSUPPORTED naming the shape (a
    shape rule: no device is needed to reach it), and the class-block entry refuses a block that wide alike."""
    L = _lib()
    lib = L.load()
    assert lib.se_linear_svm_fit(256, 4096, 64, 4096, 256, 1024, 1.0, 1e-4, 1, 256, None, None, None, 256, None) == -3
    assert '4096 x 1024 does not fit the fixed-order' in lib.se_last_error().decode()
    assert _fit_classes(L, 256, 4096, 64, 4096, 256, 3000, 1000, 1024) == -3
    assert '4096 x 1024 does not fit the fixed-order' in lib.se_last_error().decode()
