"""pairwise_distances / sinkhorn / earth_movers_distance -- the reference's names, arguments, shape rules and return
conventions (/root/reference/point_cloud_utils/_sinkhorn.py:4-156), computed by the kernels of csrc/sinkhorn.cuh.

Inputs and results take the forms of _call.py; CUDA tensors in -> CUDA tensors out, nothing synchronises.  float32 /
float64."""
import math

import numpy as _np

from . import _pcu_internal
from ._call import _asarrays, _dtype_name, _form, _run, _torch

_NORM2, _NORM1, _NORMINF, _NORMNEGINF, _NORM0, _NORMP = range(6)


def _norm_kind(p):
    if p is None or p == 2:
        return _NORM2, 2.0
    if isinstance(p, str):
        raise ValueError("Invalid norm order '%s' for vectors" % p)     # what np.linalg.norm(..., axis=-1) raises for 'fro' / 'nuc'
    if p == 1:
        return _NORM1, 1.0
    if p == math.inf:
        return _NORMINF, 0.0
    if p == -math.inf:
        return _NORMNEGINF, 0.0
    if p == 0:
        return _NORM0, 0.0
    return _NORMP, float(p)


def _float_inputs(arrays, names):
    """The form of the inputs (numpy arrays, ndarray subclasses included, or tensors) after the check of their dtype."""
    arrays = _asarrays(arrays)
    form = _form(arrays, names)
    if _dtype_name(arrays[0]) not in ("float32", "float64"):
        raise ValueError("Invalid scalar type (%s). Expected one of ['float32', 'float64']." % arrays[0].dtype)
    return form, arrays


def pairwise_distances(a, b, p=None, *, device=None):
    """
    Compute the (batched) pairwise distance matrix between a and b which both have size [m, n, d] or [n, d]. The result
    is a tensor of size [m, n, n] (or [n, n]) whose entry [m, i, j] contains the distance between a[m, i, :] and b[m, j, :].

    Args:
      a : A tensor containing m batches of n points of dimension d. i.e. of size (m, n, d)
      b : A tensor containing m batches of n points of dimension d. i.e. of size (m, n, d)
      p : Norm to use for the distance (None: the 2-norm; a number, inf, -inf or 0 as for np.linalg.norm)

    Returns:
      M : A (m, n, n)-shaped array containing the pairwise distance between each pair of inputs in a batch.

    Mirrors /root/reference/point_cloud_utils/_sinkhorn.py:4-34.
    """
    kind, pv = _norm_kind(p)
    squeezed = False
    if len(a.shape) == 2 and len(b.shape) == 2:
        a, b = a[None, :, :], b[None, :, :]
        squeezed = True
    if len(a.shape) != 3:
        raise ValueError("Invalid shape for a. Must be [m, n, d] or [n, d] but got", a.shape)
    if len(b.shape) != 3:
        raise ValueError("Invalid shape for a. Must be [m, n, d] or [n, d] but got", b.shape)
    if a.shape[0] != b.shape[0] or a.shape[2] != b.shape[2]:
        raise ValueError("operands could not be broadcast together with shapes %s %s" % (tuple(a.shape), tuple(b.shape)))
    form, (a, b) = _float_inputs([a, b], ["a", "b"])
    if b.dtype != a.dtype:
        raise ValueError("a and b must have the same dtype")
    torch = _torch()

    def body(ta, tb, dev, stream):
        nb, n, d = ta.shape
        m = tb.shape[1]
        out = torch.empty((nb, n, m), dtype=ta.dtype, device=ta.device)
        if out.numel():
            _pcu_internal._pairwise_device(ta.dtype == torch.float64, ta.data_ptr(), tb.data_ptr(), nb, n, m, d, kind, pv,
                                           out.data_ptr(), dev, stream)
        return out

    return _run(form, [a, b], device, body, squeeze=squeezed)     # np.squeeze: every size-1 dimension goes (:31-32)


def _squeeze(x):
    return _np.squeeze(x) if isinstance(x, _np.ndarray) else x.squeeze()


def sinkhorn(a, b, M, eps, max_iters=100, stop_thresh=1e-3, *, device=None, _want_cost=False):
    """
    Compute the (batched) Sinkhorn correspondences between two dirac delta distributions, U, and V.
    This implementation is numerically stable with float32.

    Args:
      a : A m-sized minibatch of weights for each dirac in the first distribution, U. i.e. shape = (m, n)
      b : A m-sized minibatch of weights for each dirac in the second distribution, V. i.e. shape = (m, n)
      M : A minibatch of n-by-n tensors storing the distance between each pair of diracs in U and V.
      eps : The reciprocal of the sinkhorn regularization parameter
      max_iters : The maximum number of Sinkhorn iterations
      stop_thresh : Stop if the change in iterates is below this value

    Returns:
      P : An (m, n, n)-shaped array of correspondences between distributions U and V

    Mirrors /root/reference/point_cloud_utils/_sinkhorn.py:37-126 (shape rules :55-99, iteration :104-118, plan :120-122).
    """
    M, a, b = _squeeze(M), _squeeze(a), _squeeze(b)
    squeezed = False
    if len(M.shape) == 2 and len(a.shape) == 1 and len(b.shape) == 1:
        M, a, b = M[None, :, :], a[None, :], b[None, :]
        squeezed = True
    elif len(M.shape) == 2 and len(a.shape) != 1:
        raise ValueError("Invalid shape for a %s, expected [m,] where m is the number of samples in a and "
                         "M has shape [m, n]" % str(tuple(a.shape)))
    elif len(M.shape) == 2 and len(b.shape) != 1:
        raise ValueError("Invalid shape for a %s, expected [m,] where n is the number of samples in a and "
                         "M has shape [m, n]" % str(tuple(b.shape)))
    if len(M.shape) != 3:
        raise ValueError("Got unexpected shape for M %s, should be [nb, m, n] where nb is batch size, and "
                         "m and n are the number of samples in the two input measures." % str(tuple(M.shape)))
    elif len(a.shape) != 2:
        raise ValueError("Invalid shape for a %s, expected [nb, m]  where nb is batch size, m is the number of samples "
                         "in a and M has shape [nb, m, n]" % str(tuple(a.shape)))
    elif len(b.shape) != 2:
        raise ValueError("Invalid shape for a %s, expected [nb, m]  where nb is batch size, m is the number of samples "
                         "in a and M has shape [nb, m, n]" % str(tuple(b.shape)))
    nb, m, n = M.shape
    if a.dtype != b.dtype or a.dtype != M.dtype:
        raise ValueError("Tensors a, b, and M must have the same dtype got: dtype(a) = %s, dtype(b) = %s, dtype(M) = %s"
                         % (str(a.dtype), str(b.dtype), str(M.dtype)))
    if tuple(a.shape) != (nb, m):
        raise ValueError("Got unexpected shape for tensor a (%s). Expected [nb, m] where M has shape [nb, m, n]." % str(tuple(a.shape)))
    if tuple(b.shape) != (nb, n):
        raise ValueError("Got unexpected shape for tensor b (%s). Expected [nb, n] where M has shape [nb, m, n]." % str(tuple(b.shape)))
    form, (a, b, M) = _float_inputs([a, b, M], ["a", "b", "M"])
    torch = _torch()

    def body(ta, tb, tM, dev, stream):
        P = torch.empty((nb, m, n), dtype=tM.dtype, device=tM.device)
        cost = torch.empty(nb, dtype=torch.float64, device=tM.device) if _want_cost else None
        _pcu_internal._sinkhorn_device(tM.dtype == torch.float64, ta.data_ptr(), tb.data_ptr(), tM.data_ptr(), nb, m, n,
                                       float(eps), int(max_iters), float(stop_thresh), P.data_ptr(),
                                       cost.data_ptr() if _want_cost else 0, 0, dev, stream)
        if squeezed:
            P = P.squeeze()
        return (P, cost) if _want_cost else P

    return _run(form, [a, b, M], device, body)


def earth_movers_distance(p, q, p_norm=2, eps=1e-4, max_iters=100, stop_thresh=1e-3, *, device=None):
    """
    Compute the (batched) Sinkhorn correspondences between two dirac delta distributions, U, and V.
    This implementation is numerically stable with float32.

    Args:
      p : An (n, d)-shaped array of d-dimensional points
      b : An (m, d)-shaped array of d-dimensional points
      p_norm : Which norm to use (default is 2),
      eps : The reciprocal of the sinkhorn regularization parameter (default 1e-4)
      max_iters : The maximum number of Sinkhorn iterations
      stop_thresh : Stop if the change in iterates is below this value

    Returns:
      emd : The earth mover's distance between point clouds p and q
      P : An (n, m)-shaped array of correspondences between point clouds p and q

    Mirrors /root/reference/point_cloud_utils/_sinkhorn.py:129-156.  Like the reference, the weights are float64
    (np.ones(n) / n): with float32 points the reference's own dtype check raises, and so does this function.
    """
    f64 = _np.float64 if isinstance(p, _np.ndarray) else getattr(_torch(), "float64")
    if p.dtype != f64 or q.dtype != f64:   # what the reference's sinkhorn() says about its own float64 weights (:88-90)
        raise ValueError("Tensors a, b, and M must have the same dtype got: dtype(a) = float64, dtype(b) = float64, dtype(M) = %s"
                         % str(p.dtype))
    M = pairwise_distances(p, q, p_norm, device=device)
    form = _form(_asarrays([p, q]), ["p", "q"])
    if form == "numpy":
        a = _np.ones(p.shape[0]) / p.shape[0]
        b = _np.ones(q.shape[0]) / q.shape[0]
    else:
        torch = _torch()
        a = torch.ones(p.shape[0], dtype=torch.float64, device=M.device) / p.shape[0]
        b = torch.ones(q.shape[0], dtype=torch.float64, device=M.device) / q.shape[0]
    P, cost = sinkhorn(a, b, M, eps, max_iters, stop_thresh, device=device, _want_cost=True)
    if form == "numpy":
        return M.dtype.type(cost.sum()), P
    return cost.sum().to(M.dtype), P
