"""Structured observation layout + device-side pack / unpack (SURVEY §8 row a-4).

Mirrors, with the same names and results:
  reference pufferlib/emulation.py:68-80    dtype_from_space   (np.dtype(..., align=True) C-struct layout)
  reference pufferlib/emulation.py:82-94    flatten_space
  reference pufferlib/emulation.py:96-112   emulate_observation_space (flat Box of the common leaf dtype / uint8)
  reference pufferlib/pytorch.py:48-100     nativize_dtype -> (torch dtype, shape, offset, delta) tree
  reference pufferlib/pytorch.py:103-145    nativize_tensor (zero-copy typed views of the flat batch)
  reference pufferlib/extensions.pyx:19-30  emulate  -> ``emulate_batch``: N samples at once on the device
                                                  (pb_struct_pack gathers the leaf tensors into C-aligned records)
  reference pufferlib/extensions.pyx:32-49  nativize -> ``nativize_batch`` (pb_struct_unpack)
The layout functions are pure host logic (numpy); the batch pack / unpack are CUDA kernels behind the C ABI.
"""
import ctypes as C

import numpy as np
import torch

from pufferlib_b200 import _native, spaces

numpy_to_torch_dtype_dict = {
    np.dtype('float64'): torch.float64, np.dtype('float32'): torch.float32, np.dtype('float16'): torch.float16,
    np.dtype('uint64'): torch.uint64, np.dtype('uint32'): torch.uint32, np.dtype('uint16'): torch.uint16,
    np.dtype('uint8'): torch.uint8, np.dtype('int64'): torch.int64, np.dtype('int32'): torch.int32,
    np.dtype('int16'): torch.int16, np.dtype('int8'): torch.int8, np.dtype('bool'): torch.bool,
}


def dtype_from_space(space):
    if isinstance(space, spaces.Tuple):
        dtype = [(f'f{i}', dtype_from_space(elem)) for i, elem in enumerate(space)]
    elif isinstance(space, spaces.Dict):
        dtype = [(k, dtype_from_space(value)) for k, value in space.items()]
    else:
        dtype = (space.dtype, space.shape)
    return np.dtype(dtype, align=True)


def flatten_space(space):
    if isinstance(space, spaces.Tuple):
        return [leaf for e in space for leaf in flatten_space(e)]
    if isinstance(space, spaces.Dict):
        return [leaf for e in space.values() for leaf in flatten_space(e)]
    return [space]


def _dtype_bounds(dtype):
    if dtype == bool:
        return 0, 1
    if np.issubdtype(dtype, np.integer):
        return np.iinfo(dtype).min, np.iinfo(dtype).max
    return np.finfo(dtype).min, np.finfo(dtype).max


def emulate_observation_space(space):
    emulated_dtype = dtype_from_space(space)
    if isinstance(space, spaces.Box):
        return space, emulated_dtype
    leaves = flatten_space(space)
    dtypes = [e.dtype for e in leaves]
    dtype = dtypes[0] if dtypes.count(dtypes[0]) == len(dtypes) else np.dtype(np.uint8)
    mmin, mmax = _dtype_bounds(dtype)
    numel = emulated_dtype.itemsize // dtype.itemsize
    return spaces.Box(low=mmin, high=mmax, shape=(numel,), dtype=dtype), emulated_dtype


def round_to(x, base):
    return int(base * np.ceil(x / base))


def _nativize_dtype(sample_dtype, structured_dtype, offset=0):
    if structured_dtype.fields is None:
        if structured_dtype.subdtype is not None:
            dtype, shape = structured_dtype.subdtype
        else:
            dtype, shape = structured_dtype, (1,)
        delta = int(np.prod(shape))
        if sample_dtype.base.itemsize == 1:
            offset = round_to(offset, dtype.alignment)
            delta *= dtype.itemsize
        else:
            assert dtype.itemsize == sample_dtype.base.itemsize
        return None, numpy_to_torch_dtype_dict[dtype], shape, offset, delta
    subviews, start_offset, all_delta = {}, offset, 0
    for name, (dtype, _) in structured_dtype.fields.items():
        views, dtype, shape, offset, delta = _nativize_dtype(sample_dtype, dtype, offset)
        subviews[name] = views if views is not None else (dtype, shape, offset, delta)
        offset += delta
        all_delta += delta
    return subviews, dtype, shape, start_offset, all_delta


def nativize_dtype(emulated):
    subviews, dtype, shape, offset, delta = _nativize_dtype(emulated.observation_dtype,
                                                            emulated.emulated_observation_dtype)
    return (dtype, shape, offset, delta) if subviews is None else subviews


def nativize_tensor(observation, native_dtype):
    """Typed zero-copy views of a flat [N, D] batch (works on CUDA tensors as-is)."""
    if isinstance(native_dtype, tuple):
        dtype, shape, offset, delta = native_dtype
        return observation.narrow(1, offset, delta).view(dtype).view(observation.shape[0], *shape)
    return {name: nativize_tensor(observation, dt) for name, dt in native_dtype.items()}


# ---- device-side batch pack / unpack -------------------------------------------------------------------------------
class Layout(C.Structure):
    _fields_ = [('n_leaves', C.c_int32), ('record_bytes', C.c_int32), ('offset', C.c_int32 * 32),
                ('nbytes', C.c_int32 * 32)]


def leaf_layout(struct_dtype):
    """Depth-first leaves of an aligned structured dtype: [(path, np dtype, shape, byte offset, byte size)]."""
    out = []

    def walk(dt, base, path):
        if dt.fields is None:
            sub, shape = dt.subdtype if dt.subdtype is not None else (dt, ())
            out.append((path, sub, tuple(shape), base, dt.itemsize))
            return
        for name, (fdt, off) in dt.fields.items():
            walk(fdt, base + off, path + (name,))
    walk(struct_dtype, 0, ())
    return out


def _c_layout(struct_dtype):
    leaves = leaf_layout(struct_dtype)
    if len(leaves) > 32:
        raise NotImplementedError('more than 32 leaves in a structured observation')
    lay = Layout(n_leaves=len(leaves), record_bytes=struct_dtype.itemsize)
    for i, (_, _, _, off, nb) in enumerate(leaves):
        lay.offset[i], lay.nbytes[i] = off, nb
    return lay, leaves


def _leaf_tensors(sample, path_list):
    def get(x, path):
        for k in path:
            x = x[int(k[1:])] if isinstance(x, (tuple, list)) else x[k]
        return x
    return [get(sample, p) for p in path_list]


def emulate_batch(struct_dtype, sample, out=None):
    """Batch form of ``emulate`` on the device: ``sample`` is the nested dict/tuple of CUDA tensors [N, *leaf shape];
    returns the uint8 record batch [N, itemsize] (padding bytes zero)."""
    lay, leaves = _c_layout(struct_dtype)
    tensors = [t.contiguous() for t in _leaf_tensors(sample, [p for p, *_ in leaves])]
    n = tensors[0].shape[0]
    for t, (_, dt, shape, _, nb) in zip(tensors, leaves):
        if t.shape[0] != n or t.numel() * t.element_size() != n * nb:
            raise ValueError('leaf tensor does not match the structured dtype')
    if out is None:
        out = torch.empty(n, struct_dtype.itemsize, dtype=torch.uint8, device=tensors[0].device)
    ptrs = (C.c_void_p * 32)(*[t.data_ptr() for t in tensors])
    _native.check(_native.lib().pb_struct_pack(C.byref(lay), ptrs, _native.ptr(out), out.stride(0), n,
                                               _native.stream_ptr()))
    return out


def nativize_batch(struct_dtype, records):
    """Inverse of ``emulate_batch``: contiguous per-leaf CUDA tensors from a record batch [N, itemsize] uint8."""
    lay, leaves = _c_layout(struct_dtype)
    n = records.shape[0]
    outs = [torch.empty((n, *shape), dtype=numpy_to_torch_dtype_dict[np.dtype(dt)], device=records.device)
            for _, dt, shape, _, _ in leaves]
    ptrs = (C.c_void_p * 32)(*[t.data_ptr() for t in outs])
    _native.check(_native.lib().pb_struct_unpack(C.byref(lay), _native.ptr(records), records.stride(0), ptrs, n,
                                                 _native.stream_ptr()))
    result = {}
    for (path, *_), t in zip(leaves, outs):
        d = result
        for k in path[:-1]:
            d = d.setdefault(k, {})
        d[path[-1] if path else ''] = t
    return result if leaves[0][0] else outs[0]
