"""The call path of the mesh-family functions: their input forms, the argument checks they share, the upload of their
inputs and the round trip from inputs to returned outputs.

numpy arrays in -> numpy out (each input is uploaded once through torch); CUDA torch tensors in -> CUDA tensors out;
CPU tensors -> CPU tensors (through numpy).  Arguments are validated, with the reference's messages, before any
device call."""
import numpy as _np

from . import _pcu_internal

_INDEX_KINDS = {"int32": 0, "int64": 1, "uint32": 2, "uint64": 3}


def _torch():
    import importlib
    return importlib.import_module("torch")


def _is_tensor(x):
    return type(x).__module__.startswith("torch")


def _dtype_name(x):
    return str(x.dtype).replace("torch.", "")


def _form(arrays, names):
    """'numpy', 'cuda' or 'cpu' (CPU tensors) for a set of inputs that must all be of one form."""
    tensors = [_is_tensor(a) for a in arrays]
    if all(tensors):
        cuda = [a.is_cuda for a in arrays]
        if all(cuda):
            if len({a.device for a in arrays}) != 1:
                raise ValueError("%s must live on one device" % ", ".join(names))
            return "cuda"
        if not any(cuda):
            return "cpu"
        raise ValueError("%s must all be CUDA tensors or all CPU tensors" % ", ".join(names))
    for a, name in zip(arrays, names):
        if type(a) != _np.ndarray:
            raise ValueError("Invalid type for %s, must be a NumPy array, but got %s." % (name, type(a)))
    return "numpy"


def _check_float(x, name):
    if _dtype_name(x) not in ("float32", "float64"):
        raise ValueError("Invalid scalar type (%s) for argument '%s'. Expected one of ['float32', 'float64']." % (_dtype_name(x), name))


def _check_index(x, name, kinds):
    if _dtype_name(x) not in kinds:
        raise ValueError("Invalid scalar type (%s) for argument '%s'. Expected one of %s." % (_dtype_name(x), name, list(kinds)))


def _check_match(x, name, ref, ref_name):
    if _dtype_name(x) != _dtype_name(ref):
        raise ValueError("Invalid scalar type (%s) for argument '%s'. Expected it to match argument '%s' which is of type %s."
                         % (_dtype_name(x), name, ref_name, _dtype_name(ref)))


def _validate_mesh(v, f, face_dtypes):
    """The binding's dtype checks, then validate_mesh (src/common/common.h:131-148)."""
    _check_float(v, "v")
    _check_index(f, "f", face_dtypes)
    vs, fs = tuple(v.shape), tuple(f.shape)
    if len(vs) != 2 or len(fs) != 2:
        raise ValueError("Only 3D inputs are supported: v and f must have shape (n, 3) and (m, 3) (n, m > 0). Got v.shape ="
                         "%s, f.shape = %s." % (vs, fs))
    if vs[0] == 0 or fs[0] == 0:
        raise ValueError("Invalid input mesh with zero elements: v and f must have shape (n, 3) and (m, 3) (n, m > 0). Got "
                         "v.shape =%s, f.shape = %s." % (vs, fs))
    if vs[1] != 3 or fs[1] != 3:
        raise ValueError("Only 3D inputs are supported: v and f must have shape (n, 3) and (m, 3) (n, m > 0). Got v.shape ="
                         "%s, f.shape = %s." % (vs, fs))


def _matrix_shape(a):
    """The (rows, cols) the reference's Eigen binding sees: a 1-D array of n elements is an (n, 1) column."""
    s = tuple(a.shape)
    return (s[0], 1) if len(s) == 1 else (s if len(s) == 2 else (int(_np.prod(s)), 1))


def _to_device(arrays, device):
    """numpy arrays -> contiguous CUDA tensors on the device= of the call (one upload each).  Unsigned index arrays
    travel as the signed type of their width (the kernels take the kind separately)."""
    from . import _dev
    torch = _torch()
    dev = _pcu_internal._current_device() if _dev(device) < 0 else _dev(device)
    signed = {"uint32": _np.int32, "uint64": _np.int64}
    return [torch.from_numpy(_np.ascontiguousarray(a).view(signed.get(a.dtype.name, a.dtype))).to(torch.device("cuda", dev))
            for a in arrays]


def _upload(form, arrays, device):
    """Contiguous CUDA tensors of the inputs, on the device of the call.  CPU tensors go through numpy."""
    from . import _same_device
    if form == "cuda":
        _same_device(arrays[0], device)
        return [a.detach().contiguous() for a in arrays]
    return _to_device([a.detach().numpy() if _is_tensor(a) else a for a in arrays], device)


def _call_args(t):
    torch = _torch()
    return t.device.index or 0, torch.cuda.current_stream(t.device).cuda_stream


def _raise_bad(bad):
    """Raises for a count (a device tensor or a host scalar) of faces with a corner out of range."""
    nbad = int(bad.item())
    if nbad:
        raise ValueError("Invalid face indices: %d faces have a corner outside [0, #v)" % nbad)


def _run(form, arrays, device, body, index=None, squeeze=False):
    """From validated inputs to the returned outputs.  body(*tensors, device index, stream) gets `arrays` as contiguous
    CUDA tensors on the device of the call; it allocates the outputs, makes the native call(s), raises the errors the
    counts it reads imply, and returns one tensor or a tuple.  squeeze: every output squeezed as npe::move squeezes
    it.  index = (array, positions): the outputs at those positions have that index array's dtype; for numpy arrays
    and CPU tensors they travelled as the signed type of its width and are viewed back as it."""
    tensors = _upload(form, arrays, device)
    out = body(*tensors, *_call_args(tensors[0]))
    single = not isinstance(out, tuple)
    out = [out] if single else list(out)
    if squeeze:
        out = [o.squeeze() for o in out]
    if form != "cuda":
        out = [o.cpu().numpy() for o in out]
        for i in index[1] if index else ():
            out[i] = out[i].view(_dtype_name(index[0]))
        if form == "cpu":
            torch = _torch()
            out = [torch.from_numpy(o) for o in out]
    return out[0] if single else tuple(out)
