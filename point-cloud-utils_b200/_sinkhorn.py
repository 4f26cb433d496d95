"""pairwise_distances / sinkhorn / earth_movers_distance -- the reference's names, arguments, shape rules and return
conventions (/root/reference/point_cloud_utils/_sinkhorn.py:4-156), computed by the kernels of csrc/sinkhorn.cuh.

numpy arrays in -> numpy arrays out (the arrays are staged on the GPU through torch, which is plumbing here: device
memory and streams); CUDA torch tensors in -> CUDA tensors out, nothing synchronises.  float32 / float64."""
import math

import numpy as _np

from . import _pcu_internal
from ._call import _torch

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


class _Staged:
    """Inputs as contiguous CUDA tensors of one dtype on one device; remembers how to hand results back."""

    def __init__(self, arrays, device):
        torch = _torch()
        self.numpy = not any(type(x).__module__.startswith("torch") for x in arrays)
        if self.numpy:
            arrs = [_np.asarray(x) for x in arrays]
            dt = arrs[0].dtype
            if dt not in (_np.float32, _np.float64):
                raise ValueError("Invalid scalar type (%s). Expected one of ['float32', 'float64']." % dt)
            dev = torch.device("cuda", _pcu_internal._current_device() if device < 0 else device)
            self.tensors = [torch.from_numpy(_np.ascontiguousarray(x)).to(dev) for x in arrs]
        else:
            if not all(isinstance(x, torch.Tensor) and x.is_cuda for x in arrays):
                raise ValueError("inputs must all be numpy arrays or all be CUDA tensors")
            if arrays[0].dtype not in (torch.float32, torch.float64):
                raise ValueError("Invalid scalar type (%s). Expected one of ['float32', 'float64']." % arrays[0].dtype)
            self.tensors = [x.detach().contiguous() for x in arrays]
        self.device = self.tensors[0].device
        self.dtype = self.tensors[0].dtype
        self.f64 = self.dtype == torch.float64
        self.stream = torch.cuda.current_stream(self.device).cuda_stream

    def out(self, t):
        return t.cpu().numpy() if self.numpy else t


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
    from . import _dev
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
    st = _Staged([a, b], _dev(device))
    ta, tb = st.tensors
    if tb.dtype != ta.dtype:
        raise ValueError("a and b must have the same dtype")
    torch = _torch()
    nb, n, d = ta.shape
    m = tb.shape[1]
    out = torch.empty((nb, n, m), dtype=st.dtype, device=st.device)
    if out.numel():
        _pcu_internal._pairwise_device(st.f64, ta.data_ptr(), tb.data_ptr(), nb, n, m, d, kind, pv, out.data_ptr(),
                                       st.device.index or 0, st.stream)
    if squeezed:
        out = out.squeeze()          # np.squeeze: every size-1 dimension goes (:31-32)
    return st.out(out)


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
    from . import _dev
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
    st = _Staged([a, b, M], _dev(device))
    ta, tb, tM = st.tensors
    torch = _torch()
    P = torch.empty((nb, m, n), dtype=st.dtype, device=st.device)
    cost = torch.empty(nb, dtype=torch.float64, device=st.device) if _want_cost else None
    _pcu_internal._sinkhorn_device(st.f64, ta.data_ptr(), tb.data_ptr(), tM.data_ptr(), nb, m, n, float(eps), int(max_iters),
                                   float(stop_thresh), P.data_ptr(), cost.data_ptr() if _want_cost else 0, 0,
                                   st.device.index or 0, st.stream)
    if squeezed:
        P = P.squeeze()
    if _want_cost:
        return st.out(P), cost, st
    return st.out(P)


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
    if isinstance(M, _np.ndarray):
        a = _np.ones(p.shape[0]) / p.shape[0]
        b = _np.ones(q.shape[0]) / q.shape[0]
    else:
        torch = _torch()
        a = torch.ones(p.shape[0], dtype=torch.float64, device=M.device) / p.shape[0]
        b = torch.ones(q.shape[0], dtype=torch.float64, device=M.device) / q.shape[0]
    P, cost, st = sinkhorn(a, b, M, eps, max_iters, stop_thresh, device=device, _want_cost=True)
    total = cost.sum()
    if st.numpy:
        return M.dtype.type(total.item()), P
    return total.to(M.dtype), P
