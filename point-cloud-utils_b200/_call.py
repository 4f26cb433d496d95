"""The package's call path: from a call's inputs, where it runs and in what form its results come back.

numpy arrays in -> numpy out (each input is uploaded once through torch, to the GPU `device=` names, else
`current_device()`); CUDA torch tensors in -> CUDA tensors out, on the device they live on (a `device=` that
contradicts it is an error); CPU tensors -> CPU tensors (through numpy).  Arguments are validated, with the reference's
messages, before any device call.  The nearest-neighbour family takes its forms, checks and device rules from here too,
but its numpy arrays and CPU tensors go to the binding's host entry points, which stage them through the library's
page-locked ring (`_numpy` in, `_as_form` out); its numpy calls never import torch."""
import numpy as _np

from . import _pcu_internal

_INDEX_KINDS = {"int32": 0, "int64": 1, "uint32": 2, "uint64": 3}


def _torch():
    import torch
    return torch


def _is_tensor(x):
    """A torch tensor (the type's module is looked at first, so that numpy inputs never import torch)."""
    return type(x).__module__.startswith("torch") and isinstance(x, _torch().Tensor)


def _dev(device):
    """``device=`` keyword -> ordinal for the native layer (-1: let the library choose, see current_device)."""
    if device is None:
        return -1
    if isinstance(device, int):
        d = device
    elif isinstance(device, str):
        name = device.strip().lower()
        if name == "cuda":
            return -1
        if not name.startswith("cuda:") or not name[5:].isdigit():
            raise ValueError("device must be an int, None, 'cuda' or 'cuda:<i>' (got %r)" % (device,))
        d = int(name[5:])
    elif getattr(device, "type", None) == "cuda":           # torch.device
        d = -1 if device.index is None else int(device.index)
    else:
        raise ValueError("device must be an int, None, 'cuda', 'cuda:<i>' or a CUDA torch.device (got %r)" % (device,))
    count = _pcu_internal._device_count()
    if d >= count or d < -1:
        raise ValueError("device %d out of range: %d usable GPU(s) visible" % (d, count))
    return d


def _ordinal(device):
    """The GPU a numpy call runs on: the one ``device=`` names, else current_device()."""
    d = _dev(device)
    return _pcu_internal._current_device() if d < 0 else d


def _same_device(t, device):
    """CUDA tensors run where they live; a contradicting device= is an argument error."""
    d = _dev(device)
    if d >= 0 and d != (t.device.index or 0):
        raise ValueError("device=%r contradicts the inputs, which live on %s" % (device, t.device))


def _call_args(t):
    """(device index, current stream) of a CUDA tensor: the last two arguments of every device entry point."""
    return t.device.index or 0, _torch().cuda.current_stream(t.device).cuda_stream


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


def _asarrays(arrays):
    """Every input that is not a tensor as np.asarray has it (ndarray subclasses such as np.memmap become arrays)."""
    return [a if _is_tensor(a) else _np.asarray(a) for a in arrays]


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


def _shape(x):
    """A shape as the reference's bindings print one: (n, 3)."""
    return "(%s)" % ", ".join(str(int(s)) for s in x.shape)


def _check_clouds(clouds, names):
    """The reference's checks of one or two point sets, in its order: the first one's dtype, the second's against it,
    then (n, 3) shapes with n > 0 (src/point_cloud_distance.cpp:133-149).  Anything with a dtype and a shape will do."""
    _check_float(clouds[0], names[0])
    for c, name in zip(clouds[1:], names[1:]):
        _check_match(c, name, clouds[0], names[0])
    shapes = [tuple(c.shape) for c in clouds]
    if all(len(s) == 2 and s[0] > 0 and s[1] == 3 for s in shapes):
        return
    got = "%s must have shape %s. Got %s." % (" and ".join(names), " and ".join(("(n, 3)", "(m, 3)")[:len(names)]),
                                             ", ".join("%s.shape = %s" % (n, _shape(c)) for c, n in zip(clouds, names)))
    if any(len(s) != 2 for s in shapes) or all(s[0] > 0 for s in shapes):
        raise ValueError("Only 3D inputs are supported: " + got)
    raise ValueError("Invalid input set with zero elements: " + got)


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


def _validate_mesh_faces(f):
    """validate_mesh_faces (src/common/common.h:112-127) on the matrix the binding sees; returns its row count."""
    rows, cols = _matrix_shape(f)
    if rows == 0:
        raise ValueError("Invalid input faces with zero elements: f must have shape (n, 3) where n > 0. Got f.shape =(%d, %d)."
                         % (rows, cols))
    if cols != 3:
        raise ValueError("Only triangle inputs are supported: f must have shape (n, 3) where n > 0. Got f.shape =(%d, %d)."
                         % (rows, cols))
    return rows


def _to_device(arrays, device):
    """numpy arrays -> contiguous CUDA tensors on the device= of the call (one upload each).  Unsigned index arrays
    travel as the signed type of their width (the kernels take the kind separately)."""
    torch = _torch()
    dev = _ordinal(device)
    signed = {"uint32": _np.int32, "uint64": _np.int64}
    return [torch.from_numpy(_np.ascontiguousarray(a).view(signed.get(a.dtype.name, a.dtype))).to(torch.device("cuda", dev))
            for a in arrays]


def _numpy(arrays):
    """The inputs as numpy arrays: CPU tensors as the arrays that share their memory."""
    return [a.detach().numpy() if _is_tensor(a) else a for a in arrays]


def _as_form(form, out):
    """Host outputs (one or a tuple) in the form of the call's inputs: for CPU tensors every array becomes a tensor,
    scalars stay as they are."""
    if form != "cpu":
        return out
    torch = _torch()
    if isinstance(out, tuple):
        return tuple(torch.from_numpy(o) if isinstance(o, _np.ndarray) else o for o in out)
    return torch.from_numpy(out) if isinstance(out, _np.ndarray) else out


def _upload(form, arrays, device):
    """Contiguous CUDA tensors of the inputs, on the device of the call.  CPU tensors go through numpy."""
    if form == "cuda":
        _same_device(arrays[0], device)
        return [a.detach().contiguous() for a in arrays]
    return _to_device(_numpy(arrays), device)


def _raise_bad(bad, message="Invalid face indices: %d faces have a corner outside [0, #v)"):
    """Raises for a count (a device tensor or a host scalar) of faces with a corner out of range, or of whatever else
    `message` names."""
    nbad = int(bad.item())
    if nbad:
        raise ValueError(message % nbad)


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
