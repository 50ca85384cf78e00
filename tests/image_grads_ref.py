"""fp64 references of the gradients the losses owe their FIRST argument (y_true), next to oracle/spec_np's closed forms
for y_pred.  Checked on CPU against fp64 autograd of oracle/ref_torch in test_image_grads_oracle.py; the GPU tests
(test_gpu_image_grads.py) hold the kernels to them."""
import numpy as np

from oracle import spec_np


def ncc_grad_true(y_true, y_pred, win=None):
    """d(-mean cc)/d(y_true), closed form in float64 (reference voxelmorph/torch/losses.py:57-67).

    With S the zero-padded box sum, n = prod(win), u_I = S(I)/n, u_J = S(J)/n the window sums reduce to
    cross = S(IJ) - S(I) S(J) / n, Ivar = S(II) - S(I)^2 / n, Jvar = S(JJ) - S(J)^2 / n, and cc = cross^2 / den with
    den = Ivar Jvar + 1e-5.  At a window p and a voxel x inside it
        d cross / dI(x) = J(x) - u_J(p),    d Ivar / dI(x) = 2 (I(x) - u_I(p)),    d Jvar / dI(x) = 0
    so  d cc / dI(x) = A (J(x) - u_J) + 2 Bp (I(x) - u_I)  with  A = 2 cross / den,  Bp = -cross^2 Jvar / den^2,
    and summing over the windows that contain x (a box sum again, the window being symmetric):
        d(sum cc)/dI = J S(A) - S(A u_J) + 2 I S(Bp) - 2 S(Bp u_I)."""
    I = np.asarray(y_true, dtype=np.float64)
    J = np.asarray(y_pred, dtype=np.float64)
    nd = I.ndim - 2
    win = [9] * nd if win is None else list(win)
    cc, t = spec_np.ncc_cc_map(I, J, win)
    den = t["Ivar"] * t["Jvar"] + 1e-5
    A = 2 * t["cross"] / den
    Bp = -(t["cross"] ** 2) * t["Jvar"] / den ** 2
    S = spec_np.box_sum
    g = J * S(A, win) - S(A * t["uJ"], win) + 2 * I * S(Bp, win) - 2 * S(Bp * t["uI"], win)
    return -g / cc.size
