"""The SHA-256 coprocessor (reference src/coprocessor/sha256.rs): its native hash and the witness of its circuit.

`synthesize_sha256` (sha256.rs:27-64) allocates, per call with n pointers: to_bits_le_strict of every pointer's tag and
hash, the aux of bellpepper's sha256 gadget over those bits, pack_bits' element and the output tag.  The library writes
that block on the GPU (include/lurk_b200.h, lurk_sha256_witness_*); the fold context writes it straight into W
(NovaFoldContext.add_sha256_batch).
"""
import hashlib

import numpy as np

from . import _capi

_NUM_BITS = {_capi.FIELD_BN254_FR: 254, _capi.FIELD_BN254_FQ: 254, _capi.FIELD_PALLAS_FQ: 255, _capi.FIELD_PALLAS_FP: 255}


class Sha256Coprocessor:
    """Sha256Coprocessor::new(n): a coprocessor of arity n"""

    def __init__(self, n):
        if n < 1:
            raise ValueError("a SHA-256 coprocessor takes at least one pointer")
        self.n = n

    def arity(self):
        return self.n

    def compute_sha256(self, field_id, ptrs):
        """sha256.rs:66-90: ptrs = n (tag, hash) pairs of field elements (ints).  SHA-256 of the pointers' 32-byte
        little-endian tag and hash, concatenated and reversed as a whole; the digest read big-endian, its top
        256 - CAPACITY bits cleared (discard_bits)."""
        if len(ptrs) != self.n:
            raise ValueError(f"{len(ptrs)} pointers for a coprocessor of arity {self.n}")
        msg = b"".join(int(t).to_bytes(32, "little") + int(h).to_bytes(32, "little") for t, h in ptrs)[::-1]
        return int.from_bytes(hashlib.sha256(msg).digest(), "big") & ((1 << (_NUM_BITS[field_id] - 1)) - 1)

    def witness_block(self, field_id):
        return witness_block(field_id, self.n)


def witness_block(field_id, n):
    """elements of the witness block of one call with n pointers"""
    size = _capi.lib().lurk_sha256_witness_block(field_id, n)
    if not size:
        raise ValueError(f"no SHA-256 witness for field {field_id} and n = {n}")
    return size


def sha256_witness_batch(field_id, n, inputs, fmt=_capi.FMT_CANONICAL):
    """inputs: uint8 array of count * 2n elements (per pointer tag, then hash) -> uint8 array of count witness blocks"""
    blk = witness_block(field_id, n)
    src = np.ascontiguousarray(inputs, dtype=np.uint8).reshape(-1)
    if src.size % (64 * n):
        raise ValueError("input buffer is not a whole number of calls")
    count = src.size // (64 * n)
    out = np.zeros(count * blk * 32, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_sha256_witness_batch(field_id, n, _capi.np_ptr(src), count, _capi.np_ptr(out), fmt))
    return out
