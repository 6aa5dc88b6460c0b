"""Linear algebra shared by the high-precision references of one Levenberg-Marquardt step (tests/pgo_reference.py,
tests/lba_reference.py): the damped system H + lambda I as a scipy.sparse matrix, its normwise backward error, an exact solve by
sparse LU with one step of iterative refinement, and an upper bound on its condition number.  H may be float64 or np.longdouble;
the backward error's residual is formed in H's precision."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl


def damped(H, lam):
    return (H + lam * sp.identity(H.shape[0], format="csc", dtype=H.dtype)).tocsc()


def backward_error(A, x, b):
    """Normwise backward error ||A x - b||_inf / (||A||_inf ||x||_inf + ||b||_inf)."""
    r = A @ x - b
    a_inf = abs(A).sum(axis=1).max()
    return float(np.abs(r).max() / (a_inf * np.abs(x).max() + np.abs(b).max()))


def factor(A):
    """Sparse LU of A (minimum degree on A^T + A, the pattern being symmetric), in float64."""
    return spl.splu(A.astype(np.float64).tocsc(), permc_spec="MMD_AT_PLUS_A")


def exact_step(A, b, lu=None):
    """A^-1 b by a sparse LU and one step of iterative refinement (the refinement residual in A's precision)."""
    lu = lu or factor(A)
    x = lu.solve(np.asarray(b, np.float64))
    return x + lu.solve(np.asarray(b - A @ x, np.float64))


def kappa_bound(A, lam):
    """Upper bound on the 2-norm condition number of A = H + lam I, H positive semi-definite: ||A||_inf (>= its largest eigenvalue)
    over lam (<= its smallest).  Lanczos takes minutes on these clustered spectra; on the 500-keyframe pose graph the bound is within
    a factor 1.3 of eigsh's condition number (tests/test_pgo_precision_cpu.py)."""
    return float(abs(A).sum(axis=1).max() / lam)


def rel(x, y):
    return float(np.linalg.norm(x - y) / np.linalg.norm(y))
