"""Host-side mirror of the reference's ntt-cuda crate (poc/ntt-cuda/src/lib.rs:20-118):
NTT / iNTT / coset_NTT / coset_iNTT, in place on a host array, through the C-ABI
`compute_ntt`-style entry points.  Element type picks the field: uint64 = Goldilocks,
uint32 = BabyBear (Montgomery words), as the reference's per-FEATURE builds do.

Input words: a Goldilocks word may be any uint64 and stands for its value mod p (non-canonical
words, as Plonky2 keeps them, are accepted); BabyBear and the 256-bit fields take canonical
Montgomery residues (< p), as the reference does.  Every entry here returns canonical words."""
import numpy as np

from . import _lib

NN, NR, RN, RR = 0, 1, 2, 3            # sppark::NTTInputOutputOrder (rust/src/lib.rs:99-105)
BB = 4                                 # extension: bit-reversed in and out (RR == NN in the reference)
FORWARD, INVERSE = 0, 1                # sppark::NTTDirection
STANDARD, COSET = 0, 1                 # sppark::NTTType
GL64, BB31 = 0, 1
BLS12_381_FR, PALLAS_FR, VESTA_FR = 2, 3, 4      # (n, 4) uint64 arrays of Montgomery residues
BN254_FR, BLS12_377_FR = 5, 6                    # likewise (domains up to 2^28 / 2^30)


def _field_of(a):
    if a.dtype == np.uint64:
        return GL64
    if a.dtype == np.uint32:
        return BB31
    raise TypeError("inout must be uint64 (Goldilocks) or uint32 (BabyBear)")


def _run(device_id, inout, order, direction, typ, field=None):
    if not isinstance(inout, np.ndarray) or not inout.flags["C_CONTIGUOUS"] or not inout.flags["WRITEABLE"]:
        raise TypeError("inout must be a writable C-contiguous numpy array")
    n = inout.size if field in (None, GL64, BB31) else inout.shape[0]
    if n & (n - 1):
        raise ValueError("inout.len() is not power of 2")     # same panic text as the crate
    lg = n.bit_length() - 1 if n else 0
    if n == 0:
        return
    field = _field_of(inout) if field is None else field
    l = _lib.lib()
    if field == GL64:
        err = l.compute_ntt(device_id, inout.ctypes.data, lg, order, direction, typ)
    else:
        err = l.sppark_b200_ntt(field, device_id, inout.ctypes.data, lg, order, direction, typ)
    _lib.check(err)


def NTT(device_id, inout, order=NN, field=None):
    _run(device_id, inout, order, FORWARD, STANDARD, field)


def iNTT(device_id, inout, order=NN, field=None):
    _run(device_id, inout, order, INVERSE, STANDARD, field)


def coset_NTT(device_id, inout, order=NN, field=None):
    _run(device_id, inout, order, FORWARD, COSET, field)


def coset_iNTT(device_id, inout, order=NN, field=None):
    _run(device_id, inout, order, INVERSE, COSET, field)


def LDE(device_id, evals, lg_blowup, field=None, want_coefficients=False):
    """NTT::LDE (ntt/ntt.cuh:336-338): evaluations on the 2^lg domain -> evaluations on the coset
    of the 2^(lg+lg_blowup) domain (natural order).  Returns the extended array (and the natural
    -order coefficients if asked, as LDE_aux does)."""
    field = _field_of(evals) if field is None else field
    n = evals.size if field in (GL64, BB31) else evals.shape[0]
    if n & (n - 1):
        raise ValueError("inout.len() is not power of 2")
    lg = n.bit_length() - 1
    shape = (n << lg_blowup,) + tuple(evals.shape[1:])
    ext = np.zeros(shape, dtype=evals.dtype)
    ext[:n] = evals
    aux = np.zeros_like(evals) if want_coefficients else None
    err = _lib.lib().sppark_b200_lde(field, device_id, ext.ctypes.data, lg, lg_blowup,
                                     aux.ctypes.data if aux is not None else None)
    _lib.check(err)
    return (ext, aux) if want_coefficients else ext


def ntt_dev(tensor, order=NN, direction=FORWARD, typ=STANDARD, field=None, stream=None):
    """NTT::Base_dev_ptr (ntt/ntt.cuh:344-350): in place on a CUDA torch tensor, enqueued on
    torch's current stream (or `stream`), not synchronised."""
    import torch
    assert tensor.is_cuda and tensor.is_contiguous()
    n = tensor.numel()
    if n & (n - 1):
        raise ValueError("inout.len() is not power of 2")
    if field is None:
        field = {8: GL64, 4: BB31}[tensor.element_size()]
    with torch.cuda.device(tensor.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_ntt_dev(field, tensor.data_ptr(), n.bit_length() - 1,
                                             order, direction, typ, s)
    _lib.check(err)


def _batch_shape(shape, itemsize, field):
    """(batch, n) for the one-word fields, (batch, n, 4) uint64 words for the 256-bit fields; the
    element size must be the field's word size, or the library would run past the buffer"""
    wide = field not in (GL64, BB31)
    if itemsize != (4 if field == BB31 else 8):
        raise ValueError(f"{itemsize}-byte elements do not match field {field}")
    if len(shape) != (3 if wide else 2) or (wide and shape[2] != 4):
        raise ValueError("batched arrays are (batch, n)" + (", 4) uint64 for this field" if wide else ""))
    batch, n = int(shape[0]), int(shape[1])
    if n == 0 or n & (n - 1):
        raise ValueError("row length is not a power of 2")
    return batch, n.bit_length() - 1


def ntt_batch(device_id, inout, order=NN, direction=FORWARD, typ=STANDARD, field=None):
    """`batch` same-size transforms in one call, in place on a host array: row b of a C-contiguous
    (batch, n) array (or (batch, n, 4) uint64 for the 256-bit fields) comes out as
    NTT/iNTT/coset_* would return it alone.  Synchronised."""
    if not isinstance(inout, np.ndarray) or not inout.flags["C_CONTIGUOUS"] or not inout.flags["WRITEABLE"]:
        raise TypeError("inout must be a writable C-contiguous numpy array")
    field = _field_of(inout) if field is None else field
    batch, lg = _batch_shape(inout.shape, inout.itemsize, field)
    _lib.check(_lib.lib().sppark_b200_ntt_batch(field, device_id, inout.ctypes.data, lg, batch,
                                                order, direction, typ))


def _dev_field(tensor, field):
    if field is None:
        if tensor.element_size() not in (4, 8):
            raise ValueError("tensor elements must be 8 bytes (Goldilocks) or 4 bytes (BabyBear)")
        field = {8: GL64, 4: BB31}[tensor.element_size()]
    return field


def ntt_batch_dev(tensor, order=NN, direction=FORWARD, typ=STANDARD, field=None, stream=None):
    """ntt_batch on a CUDA torch tensor of the same shapes: in place, enqueued on torch's current
    stream (or `stream`), not synchronised."""
    import torch
    if not tensor.is_cuda or not tensor.is_contiguous():
        raise ValueError("tensor must be a contiguous CUDA tensor")
    field = _dev_field(tensor, field)
    batch, lg = _batch_shape(tuple(tensor.shape), tensor.element_size(), field)
    with torch.cuda.device(tensor.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_ntt_batch_dev(field, tensor.data_ptr(), lg, batch, order, direction, typ, s)
    _lib.check(err)


def lde_batch_dev(d_in, lg_blowup, field=None, stream=None):
    """LDE of every row of a (batch, n) CUDA tensor (or (batch, n, 4) for the 256-bit fields):
    returns a new (batch, n << lg_blowup) tensor whose rows are what LDE returns for each row,
    and leaves each row's coefficients, in bit-reversed order, in d_in.  Enqueued on torch's
    current stream (or `stream`), not synchronised."""
    import torch
    if not d_in.is_cuda or not d_in.is_contiguous():
        raise ValueError("d_in must be a contiguous CUDA tensor")
    field = _dev_field(d_in, field)
    batch, lg = _batch_shape(tuple(d_in.shape), d_in.element_size(), field)
    out = torch.empty((batch, (1 << lg) << lg_blowup) + tuple(d_in.shape[2:]), dtype=d_in.dtype, device=d_in.device)
    with torch.cuda.device(d_in.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_lde_batch_dev(field, out.data_ptr(), d_in.data_ptr(), lg, lg_blowup, batch, s)
    _lib.check(err)
    return out


def _matrix_shape(shape, itemsize, field):
    """(lg, width) of a (2^lg, width) matrix of Goldilocks (8-byte) or BabyBear (4-byte) words; the
    element size must be the field's word size, or the library would run past the buffer"""
    if field not in (GL64, BB31):
        raise ValueError(f"field {field}: the matrix entries serve Goldilocks and BabyBear only")
    if itemsize != (4 if field == BB31 else 8):
        raise ValueError(f"{itemsize}-byte elements do not match field {field}")
    if len(shape) != 2:
        raise ValueError("matrices are (2^lg, width) arrays")
    n, width = int(shape[0]), int(shape[1])
    if n == 0 or n & (n - 1):
        raise ValueError("matrix height is not a power of 2")
    return n.bit_length() - 1, width


def ntt_matrix(device_id, inout, order=NN, direction=FORWARD, typ=STANDARD, field=None):
    """The transform down every column of a writable C-contiguous (2^lg, width) array (uint64 =
    Goldilocks, uint32 = BabyBear), in place: column c comes out as NTT/iNTT/coset_* would return it
    alone.  No transpose is made.  Synchronised."""
    if not isinstance(inout, np.ndarray) or not inout.flags["C_CONTIGUOUS"] or not inout.flags["WRITEABLE"]:
        raise ValueError("inout must be a writable C-contiguous numpy array")
    if field is None:
        if inout.dtype not in (np.uint64, np.uint32):
            raise ValueError("inout must be uint64 (Goldilocks) or uint32 (BabyBear)")
        field = _field_of(inout)
    lg, width = _matrix_shape(inout.shape, inout.itemsize, field)
    _lib.check(_lib.lib().sppark_b200_ntt_matrix(field, device_id, inout.ctypes.data, lg, width,
                                                 order, direction, typ))


def ntt_matrix_dev(tensor, order=NN, direction=FORWARD, typ=STANDARD, field=None, stream=None):
    """ntt_matrix on a contiguous (2^lg, width) CUDA torch tensor: in place, enqueued on torch's
    current stream (or `stream`), not synchronised."""
    import torch
    if not tensor.is_cuda or not tensor.is_contiguous():
        raise ValueError("tensor must be a contiguous CUDA tensor")
    field = _dev_field(tensor, field)
    lg, width = _matrix_shape(tuple(tensor.shape), tensor.element_size(), field)
    with torch.cuda.device(tensor.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_ntt_matrix_dev(field, tensor.data_ptr(), lg, width, order, direction, typ, s)
    _lib.check(err)


def lde_matrix_dev(d_in, lg_blowup, field=None, stream=None):
    """LDE of every column of a contiguous (2^lg, width) CUDA tensor: returns a new
    (2^(lg + lg_blowup), width) tensor whose column c is what LDE returns for column c, and leaves
    each column's coefficients, in bit-reversed row order, in d_in.  Enqueued on torch's current
    stream (or `stream`), not synchronised."""
    import torch
    if not d_in.is_cuda or not d_in.is_contiguous():
        raise ValueError("d_in must be a contiguous CUDA tensor")
    field = _dev_field(d_in, field)
    lg, width = _matrix_shape(tuple(d_in.shape), d_in.element_size(), field)
    out = torch.empty(((1 << lg) << lg_blowup, width), dtype=d_in.dtype, device=d_in.device)
    with torch.cuda.device(d_in.device):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        err = _lib.lib().sppark_b200_lde_matrix_dev(field, out.data_ptr(), d_in.data_ptr(), lg, lg_blowup, width, s)
    _lib.check(err)
    return out
