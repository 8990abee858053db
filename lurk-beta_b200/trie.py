"""Host-side mirror of the sparse Poseidon trie of the trie coprocessor (reference src/coprocessor/trie/mod.rs), backed by
the CUDA Poseidon kernels through `PoseidonCache`.

`StandardTrie = Trie<F, 8, 85>` (trie/mod.rs:43): arity 8, height 85 (3 x 85 = 255 key bits), empty element 0.  Same
method names as the reference: `path` (mod.rs:589-609), `empty_root` (485-497), `lookup` / `lookup_aux` (635-652),
`insert` (745-776), `prove_lookup_at_path` (725-743).  The evaluation side hashes through
`PoseidonCache::compute_hash` (hash.rs:97-113) and records preimages in an inverse cache, exactly like the reference;
`lookup_circuit_witnesses` produces the 85 arity-8 slot witnesses the lookup circuit allocates (SURVEY.md 8(a) a12) in
ONE batched launch -- the 85 hashes of a path are independent once the preimages are known.

The lookup and insert circuits' whole aux blocks (synthesize_lookup_aux, mod.rs:118-156; synthesize_insert_aux,
226-268) are written on the GPU from the calls' proofs (`prove_lookup` / `prove_insert`, mod.rs:718-776):
`lookup_inputs` / `insert_inputs` pack a call, `trie_witness_batch` writes the blocks (include/lurk_b200.h,
lurk_trie_witness_*), and the fold context writes them straight into W (NovaFoldContext.add_trie_batch)."""
import ctypes as C
from collections import namedtuple

import numpy as np

from . import _capi
from .hash import PoseidonCache
from .slots import SlotType, slot_witness_batch_bytes
from .field import pack, unpack

TRIE_LOOKUP, TRIE_INSERT = _capi.TRIE_LOOKUP, _capi.TRIE_INSERT
LookupProof = namedtuple("LookupProof", "preimage_path")            # root level first, ARITY elements each
InsertProof = namedtuple("InsertProof", "old_proof new_proof")      # LookupProofs before and after the insert


class Trie:
    def __init__(self, poseidon_cache=None, arity=8, height=85, root=None, inverse_cache=None):
        if arity & (arity - 1):
            raise ValueError("ARITY must be a power of two")          # checked in new_aux()
        self.hash_cache = poseidon_cache or PoseidonCache()
        self.arity, self.height = arity, height
        self.children = inverse_cache if inverse_cache is not None else {}   # digest -> preimage (InversePoseidonCache)
        self.empty_roots = []
        cur = self.empty_element()
        for _ in range(height):
            cur = self.register_hash([cur] * arity)
            self.empty_roots.append(cur)
        self.root = self.empty_roots[height - 1] if root is None else int(root)

    @staticmethod
    def empty_element():
        return 0

    def register_hash(self, preimage):
        d = self.hash_cache.compute_hash(list(preimage))
        self.children[d] = tuple(int(x) for x in preimage)
        return d

    def empty_root_for_height(self, height):
        return self.empty_element() if height == 0 else self.empty_roots[height - 1]

    def empty_root(self):
        return self.empty_root_for_height(self.height)

    def arity_bits(self):
        return self.arity.bit_length() - 1

    def path(self, key):
        """most-significant chunk first, `arity_bits` bits per level (mod.rs:589-609)"""
        ab, n = self.arity_bits(), self.height
        key = int(key)
        return [(key >> (ab * (n - 1 - i))) & (self.arity - 1) for i in range(n)]

    def prove_lookup_at_path(self, path):
        preimages, nxt = [], self.root
        for k in path:
            if nxt not in self.children:
                raise KeyError(f"MissingPreimage({hex(nxt)})")
            pre = self.children[nxt]
            preimages.append(pre)
            nxt = pre[k]
        return preimages

    def prove_lookup(self, key):
        """the preimages on the key's path, root level first; the last one holds the payload (mod.rs:718-743)"""
        return LookupProof(self.prove_lookup_at_path(self.path(key)))

    def prove_insert(self, key, value):
        """insert and return (InsertProof(old, new), inserted): the path's preimages before and after (mod.rs:751-811)"""
        path = self.path(key)
        old = self.prove_lookup_at_path(path)
        value = int(value)
        new = []
        for k, existing in zip(reversed(path), reversed(old)):
            new_pre = list(existing)
            new_pre[k] = value
            value = self.register_hash(new_pre)
            new.append(tuple(new_pre))
        new.reverse()
        inserted = value != self.root
        self.root = value
        return InsertProof(LookupProof(old), LookupProof(new)), inserted

    def lookup_aux(self, key):
        path = self.path(key)
        return self.prove_lookup_at_path(path)[-1][path[-1]]

    def lookup(self, key):
        v = self.lookup_aux(key)
        return None if v == self.empty_element() else v

    def insert(self, key, value):
        return self.prove_insert(key, value)[1]

    def lookup_circuit_witnesses(self, key, fmt=0):
        """the HEIGHT arity-8 Poseidon witnesses of synthesize_lookup (mod.rs:654-724) as one batch: uint8 array of
        HEIGHT slot blocks, root level first"""
        preimages = self.prove_lookup_at_path(self.path(key))
        st = {4: SlotType.Hash4, 8: SlotType.Hash8}[self.arity]
        return slot_witness_batch_bytes(self.hash_cache.field_id, st, pack([x for p in preimages for x in p]), fmt)


def StandardTrie(poseidon_cache=None, root=None, inverse_cache=None):
    return Trie(poseidon_cache, 8, 85, root, inverse_cache)


def lookup_inputs(root, key, proof):
    """one lookup call's inputs: root, key, the proof's preimages root level first (2 + 8H elements, ints)"""
    return [int(root), int(key)] + [int(x) for pre in proof.preimage_path for x in pre]


def insert_inputs(root, key, value, proof):
    """one insert call's inputs: the root before the insert, key, value, the old path, the new path (3 + 16H elements)"""
    return ([int(root), int(key), int(value)] + [int(x) for pre in proof.old_proof.preimage_path for x in pre]
            + [int(x) for pre in proof.new_proof.preimage_path for x in pre])


def trie_n_inputs(op, height):
    return 3 + 16 * height if op == TRIE_INSERT else 2 + 8 * height


def trie_witness_block(field_id, op, height):
    """elements of the witness block of one lookup (op TRIE_LOOKUP) or insert (TRIE_INSERT) call at this height"""
    size = _capi.lib().lurk_trie_witness_block(field_id, op, height)
    if not size:
        raise ValueError(f"no trie witness for field {field_id}, op {op} and height {height}")
    return size


def trie_witness_batch(field_id, op, height, inputs, fmt=_capi.FMT_CANONICAL):
    """inputs: uint8 array of count calls' inputs (lookup_inputs / insert_inputs, packed) -> uint8 array of count
    witness blocks.  Raises LurkError (ERR_ARG, naming the call and level) when a call's paths do not chain."""
    blk = trie_witness_block(field_id, op, height)
    src = np.ascontiguousarray(inputs, dtype=np.uint8).reshape(-1)
    per = 32 * trie_n_inputs(op, height)
    if src.size % per:
        raise ValueError("input buffer is not a whole number of calls")
    count = src.size // per
    out = np.zeros(count * blk * 32, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_trie_witness_batch(field_id, op, height, _capi.np_ptr(src), count, _capi.np_ptr(out), fmt))
    return out


class DeviceTrie:
    """A trie node store on the GPU (include/lurk_b200.h, lurk_trie_ctx_*): arity 8, height 1..85, one field.  `apply`
    runs a batch of lookups and inserts in program order, exactly as the sequential `Trie` would, and writes every
    call's proof in `lookup_inputs` / `insert_inputs` layout to device memory, ready for the witness kernels."""

    def __init__(self, field_id=_capi.FIELD_BN254_FR, height=85, capacity=1 << 20):
        self.field_id, self.height = field_id, height
        self._lib = _capi.lib()
        # the store is built on the CUDA device current at creation (torch's, once torch has made its context current):
        # the _dev calls take tensors on that device only
        self._device = None
        if self._lib.lurk_device_count() > 0:
            import torch
            if torch.cuda.is_available():
                self._device = torch.cuda.current_device()
        ctx = C.c_void_p()
        _capi.check(self._lib.lurk_trie_ctx_create(field_id, height, capacity, C.byref(ctx)))
        self._ctx = ctx

    def close(self):
        if self._ctx:
            self._lib.lurk_trie_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def empty_root(self, fmt=_capi.FMT_CANONICAL):
        out = np.zeros(32, dtype=np.uint8)
        _capi.check(self._lib.lurk_trie_ctx_empty_root(self._ctx, _capi.np_ptr(out), fmt))
        return unpack(out)[0]

    @property
    def node_count(self):
        n, cap = C.c_uint64(), C.c_uint64()
        _capi.check(self._lib.lurk_trie_ctx_info(self._ctx, C.byref(n), C.byref(cap)))
        return n.value

    @property
    def capacity(self):
        n, cap = C.c_uint64(), C.c_uint64()
        _capi.check(self._lib.lurk_trie_ctx_info(self._ctx, C.byref(n), C.byref(cap)))
        return cap.value

    def register(self, preimages, fmt=_capi.FMT_CANONICAL):
        """add existing nodes (8-tuples of ints, e.g. a host `Trie`'s inverse cache values) -> their digests"""
        pre = pack([int(x) for p in preimages for x in p])
        if pre.size % (32 * 8):
            raise ValueError("preimages must have 8 elements each")
        n = pre.size // (32 * 8)
        out = np.zeros(n * 32, dtype=np.uint8)
        _capi.check(self._lib.lurk_trie_ctx_register(self._ctx, _capi.np_ptr(pre), n, _capi.np_ptr(out), fmt))
        return unpack(out)

    def apply(self, ops, fmt=_capi.FMT_CANONICAL, lookup_out=None, insert_out=None, stream=None):
        """ops: sequence of (kind, prev, root, key, value), ints (root read where prev = -1, value for inserts).
        Returns (results, lookup_inputs, insert_inputs): results a list of ints (lookup: the value, 0 when absent;
        insert: the new root), the proofs as uint8 CUDA tensors of (lookups, 2 + 8H, 32) and (inserts, 3 + 16H, 32)
        elements in fmt.  lookup_out / insert_out: device buffers (torch tensors) to write the proofs into instead."""
        import torch
        n = len(ops)
        kinds = np.array([o[0] for o in ops], dtype=np.int32)
        prev = np.array([o[1] for o in ops], dtype=np.int64)
        roots, keys, vals = (pack([int(o[k]) for o in ops]) if n else np.zeros(0, dtype=np.uint8) for k in (2, 3, 4))
        n_ins = int((kinds == TRIE_INSERT).sum())
        H = self.height
        if lookup_out is None:
            lookup_out = torch.empty((n - n_ins, trie_n_inputs(TRIE_LOOKUP, H), 32), dtype=torch.uint8, device="cuda")
        if insert_out is None:
            insert_out = torch.empty((n_ins, trie_n_inputs(TRIE_INSERT, H), 32), dtype=torch.uint8, device="cuda")
        for out, op, count in ((lookup_out, TRIE_LOOKUP, n - n_ins), (insert_out, TRIE_INSERT, n_ins)):
            want = count * trie_n_inputs(op, H) * 32
            if out.dtype != torch.uint8 or not out.is_cuda or not out.is_contiguous() or out.numel() != want:
                raise ValueError(f"the {'lookup' if op == TRIE_LOOKUP else 'insert'} proofs need a contiguous uint8 CUDA tensor of "
                                 f"{want} bytes, not {out.dtype} on {out.device} with {out.numel()} elements")
        res = np.zeros(n * 32, dtype=np.uint8)
        if stream is None:
            stream = torch.cuda.current_stream().cuda_stream
        _capi.check(self._lib.lurk_trie_ctx_apply(self._ctx, n, _capi.np_ptr(kinds), _capi.np_ptr(prev), _capi.np_ptr(roots), _capi.np_ptr(keys),
                                                  _capi.np_ptr(vals), fmt, _capi.np_ptr(res), lookup_out.data_ptr() if lookup_out.numel() else None,
                                                  insert_out.data_ptr() if insert_out.numel() else None, stream))
        return unpack(res), lookup_out, insert_out

    def register_dev(self, preimages, fmt=_capi.FMT_CANONICAL, digests_out=None, stream=None):
        """`register` on device memory: preimages a contiguous uint8 CUDA tensor of (n, 8, 32), elements in fmt.
        Returns the digests as a uint8 CUDA tensor of (n, 32) in fmt (digests_out when given)."""
        import torch
        _check_dev("preimages", preimages, torch.uint8, 3)
        n = preimages.shape[0]
        if tuple(preimages.shape[1:]) != (8, 32):
            raise ValueError(f"preimages must be (n, 8, 32), not {tuple(preimages.shape)}")
        if digests_out is not None:
            _check_dev("digests_out", digests_out, torch.uint8, 2, (n, 32))
        self._on_store_device(preimages=preimages, digests_out=digests_out)
        st = _call_stream(torch, stream, preimages.device)
        with torch.cuda.stream(st):
            if digests_out is None:
                digests_out = torch.empty((n, 32), dtype=torch.uint8, device=preimages.device)
        _capi.check(self._lib.lurk_trie_ctx_register_dev(self._ctx, _dptr(preimages), n, _dptr(digests_out), fmt, st.cuda_stream))
        return digests_out

    def apply_dev(self, kinds, prev, roots, keys, values, fmt=_capi.FMT_CANONICAL, results=None, lookup_out=None, insert_out=None, stream=None):
        """`apply` on operations already in device memory, planned on the GPU: kinds int32 (n,), prev int64 (n,), roots /
        keys / values uint8 (n, 32) in fmt, all contiguous CUDA tensors; roots or values may be None when never read.
        Returns (results, lookup_inputs, insert_inputs) as uint8 CUDA tensors of (n, 32), (lookups, 2 + 8H, 32) and
        (inserts, 3 + 16H, 32), in fmt; results / lookup_out / insert_out: caller tensors to write into instead, of exactly
        the batch's size.  stream: the CUDA stream handle the call is ordered on (default: torch's current stream); the
        batch's insert count, which sizes the proof buffers, is read on that stream too, after the caller's work there."""
        import torch
        _check_dev("kinds", kinds, torch.int32, 1)
        n = kinds.shape[0]
        _check_dev("prev", prev, torch.int64, 1, (n,))
        _check_dev("keys", keys, torch.uint8, 2, (n, 32))
        for name, t in (("roots", roots), ("values", values)):
            if t is not None:
                _check_dev(name, t, torch.uint8, 2, (n, 32))
        for name, t in (("results", results), ("lookup_out", lookup_out), ("insert_out", insert_out)):
            if t is not None:
                _check_dev(name, t, torch.uint8, 2 if name == "results" else None, (n, 32) if name == "results" else None)
        self._on_store_device(kinds=kinds, prev=prev, roots=roots, keys=keys, values=values, results=results, lookup_out=lookup_out,
                              insert_out=insert_out)
        H, dev = self.height, kinds.device
        st = _call_stream(torch, stream, dev)
        with torch.cuda.stream(st):
            # the proofs are written at rank x proof size: every buffer must hold exactly the batch's lookups or inserts
            n_ins = int((kinds == TRIE_INSERT).sum())
            if results is None:
                results = torch.empty((n, 32), dtype=torch.uint8, device=dev)
            if lookup_out is None:
                lookup_out = torch.empty((n - n_ins, trie_n_inputs(TRIE_LOOKUP, H), 32), dtype=torch.uint8, device=dev)
            if insert_out is None:
                insert_out = torch.empty((n_ins, trie_n_inputs(TRIE_INSERT, H), 32), dtype=torch.uint8, device=dev)
        for name, out, op, count in (("lookup_out", lookup_out, TRIE_LOOKUP, n - n_ins), ("insert_out", insert_out, TRIE_INSERT, n_ins)):
            want = count * trie_n_inputs(op, H) * 32
            if out.numel() != want:
                raise ValueError(f"{name} must hold the batch's {count} proofs of {trie_n_inputs(op, H)} elements ({want} bytes), "
                                 f"not {out.numel()} bytes")
        _capi.check(self._lib.lurk_trie_ctx_apply_dev(self._ctx, n, _dptr(kinds), _dptr(prev), _dptr(roots), _dptr(keys), _dptr(values), fmt,
                                                      _dptr(results), _dptr(lookup_out), _dptr(insert_out), st.cuda_stream))
        return results, lookup_out, insert_out

    def _on_store_device(self, **tensors):
        """every tensor given is on a CUDA device, the one the store was built on, else ValueError"""
        _on_cuda(**tensors)
        for name, t in tensors.items():
            if t is not None and self._device is not None and t.device.index != self._device:
                raise ValueError(f"{name} is on {t.device}, but the trie store was built on cuda:{self._device}")


def _call_stream(torch, stream, device):
    """the torch stream of a call: torch's current one on the device, or the caller's handle"""
    current = torch.cuda.current_stream(device)
    if stream is None or int(stream) == current.cuda_stream:
        return current
    return torch.cuda.ExternalStream(int(stream), device=device)


def _dptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def _check_dev(name, t, dtype, ndim, shape=None):
    """a contiguous tensor of this dtype (and rank and shape when given), else ValueError; _on_cuda checks the device"""
    import torch
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a CUDA tensor, not {type(t).__name__}")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, not {t.dtype}")
    if (ndim is not None and t.dim() != ndim) or (shape is not None and tuple(t.shape) != tuple(shape)):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, not {tuple(shape) if shape is not None else f'{ndim} dimensions'}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def _on_cuda(**tensors):
    """every tensor given (None: not given) is on one CUDA device, else ValueError"""
    devices = set()
    for name, t in tensors.items():
        if t is None:
            continue
        if not t.is_cuda:
            raise ValueError(f"{name} must be on a CUDA device, not {t.device}")
        devices.add(t.device)
    if len(devices) > 1:
        raise ValueError(f"the tensors are on more than one device: {sorted(str(d) for d in devices)}")


def write_trie_batch(device_trie, fold_ctx, b, batch_index, ops):
    """apply `ops` (all lookups or all inserts, the op of the NovaFoldContext's trie batch `batch_index`; for a
    SuperNovaFoldContext pass the circuit's context, `contexts[i]`) and write their proofs, Montgomery form, straight
    into the batch's device buffer of buffer set b, for stage_a(b, resident=True).  ops as for DeviceTrie.apply, in
    canonical ints; returns the results as canonical ints."""
    import torch
    kinds = {int(o[0]) for o in ops}
    if len(kinds) > 1:
        raise ValueError("a trie batch holds calls of one op")
    op = kinds.pop() if kinds else TRIE_LOOKUP
    # the library refuses elements >= p; here they must be refused before the conversion reduces them
    p = int.from_bytes(_modulus(device_trie.field_id), "little")
    for i, (_, prev, root, key, value) in enumerate(ops):
        for name, x, read in (("root", root, prev < 0), ("key", key, True), ("value", value, op == TRIE_INSERT)):
            if read and not 0 <= int(x) < p:
                raise ValueError(f"trie operation {i}: the {name} is not reduced below the field modulus")
    view = fold_ctx.device_view(b, batch_index)
    per = trie_n_inputs(op, device_trie.height) * 32
    if view.numel() != per * len(ops):
        raise ValueError(f"the batch's device buffer holds {view.numel() // per} calls, not {len(ops)}")
    out = view.view(len(ops), -1, 32)
    empty = torch.empty((0, 1, 32), dtype=torch.uint8, device="cuda")
    r_mont, r_inv = (1 << 256) % p, pow(1 << 256, -1, p)
    mont = [(k, prev, int(root) * r_mont % p, int(key) * r_mont % p, int(value) * r_mont % p) for k, prev, root, key, value in ops]
    res, _, _ = device_trie.apply(mont, fmt=_capi.FMT_MONTGOMERY, lookup_out=out if op == TRIE_LOOKUP else empty,
                                  insert_out=out if op == TRIE_INSERT else empty)
    return [r * r_inv % p for r in res]


def _modulus(field_id):
    out = np.zeros(32, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_field_modulus(field_id, _capi.np_ptr(out)))
    return out.tobytes()
