"""The linear-SVM workspace at every size (tests only): svm_oracle.svm_layout extended by the GEMM row blocks.

Where Np x Dp or Np x Cp reaches 2^31, csrc/linear_svm.cu cuts the rows into nblk equal blocks of rb rows (a multiple of
the hinge pass's 64), each GEMM call taking fewer than 2^31 elements of X, S and R, and pads Np to nblk * rb; every
region keeps its order and 256-byte alignment.  Below that size the layout is svm_oracle.svm_layout's, unchanged."""
import svm_oracle

GEMM_ELEMS = 1 << 31


def row_blocks(N, D, C):
    """(Np, rb, nblk) of the solver's GEMM row blocks."""
    up = lambda v, a: (v + a - 1) // a * a
    Np, Dp, Cp = max(N, 32), up(D, 4), up(C, 16)
    wide = max(Dp, Cp)
    if Np * wide < GEMM_ELEMS:
        return Np, Np, 1
    rb_max = (GEMM_ELEMS - 1) // wide // svm_oracle.SVM_HB_ROWS * svm_oracle.SVM_HB_ROWS
    nblk = (Np + rb_max - 1) // rb_max
    rb = up((Np + nblk - 1) // nblk, svm_oracle.SVM_HB_ROWS)
    return rb * nblk, rb, nblk


def svm_layout(N, D, C):
    """(dims, regions, total bytes) as svm_oracle.svm_layout, with dims['rb'] and dims['nblk'] added."""
    up = lambda v, a: (v + a - 1) // a * a
    Np, rb, nblk = row_blocks(N, D, C)
    Dp, Cp = up(D, 4), up(C, 16)
    P, nrb = Dp + 1, (Np + svm_oracle.SVM_HB_ROWS - 1) // svm_oracle.SVM_HB_ROWS
    dims = dict(N=N, Np=Np, Dp=Dp, P=P, C=C, Cp=Cp, nrb=nrb, rb=rb, nblk=nblk)
    regions = [('xp', (Np, Dp), 'f4'), ('s_cur', (Np, Cp), 'f4'), ('s_trial', (Np, Cp), 'f4'), ('R', (Np, Cp), 'f4')]
    regions += [(v, (P, Cp), 'f4') for v in svm_oracle.SVM_VECTORS]
    regions += [('partial', (nrb, Cp), 'f8'), ('state', (Cp,), 'state'), ('counts', (Cp + 1,), 'i4'), ('ctr', (4,), 'i4')]
    size = {'f4': 4, 'f8': 8, 'state': 128, 'i4': 4}
    out, o = [], 0
    for name, shape, kind in regions:
        out.append((name, o, shape, kind))
        n = 1
        for s in shape:
            n *= s
        o = up(o + n * size[kind], 256)
    return dims, out, o


def workspace_views(ws, N, D, C):
    """svm_oracle.svm_workspace_views on the extended layout."""
    import torch
    _, regions, total = svm_layout(N, D, C)
    assert ws.numel() >= total
    dt = {'f4': torch.float32, 'f8': torch.float64, 'i4': torch.int32, 'state': torch.uint8}
    out = {}
    for name, off, shape, kind in regions:
        n = 1
        for s in shape:
            n *= s
        nb = n * (128 if kind == 'state' else torch.tensor([], dtype=dt[kind]).element_size())
        out[name] = ws[off:off + nb].view(dt[kind]).view(*shape) if kind != 'state' else ws[off:off + nb]
    return out
