"""Host-side mirror of the fold context of liblurk_b200 (include/lurk_b200.h, S5/S6): the GPU half of
`Proof::prove_recursively` (reference src/proof/nova.rs:260-339, supernova.rs:207-291).

The schedule itself -- stage A of later steps on its own streams, the sequential chain of stage B without host round
trips, the exchange of partial commitments between GPUs, the random-oracle challenge -- lives in the library
(csrc/foldctx_impl.cuh); this module only marshals buffers.  `NovaFoldContext` is one running instance (one circuit);
`SuperNovaFoldContext` holds one per circuit index (NIVC, src/lem/multiframe.rs:941).
"""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import (FOLD_BUF_E1, FOLD_BUF_GLUE, FOLD_BUF_RO, FOLD_BUF_T, FOLD_BUF_W2, FOLD_BUF_X2, FOLD_BUF_Z1, FOLD_INPUTS_RESIDENT,
                    FoldConfig, FoldResult, FoldSpan)


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8).reshape(-1)


class StepResult:
    """record of one step: 96-byte points x|y|z and 32-byte elements, in the format asked for"""

    def __init__(self, raw):
        self.comm_W = np.frombuffer(bytes(raw.comm_W), dtype=np.uint8).copy()
        self.comm_T = np.frombuffer(bytes(raw.comm_T), dtype=np.uint8).copy()
        self.r = np.frombuffer(bytes(raw.r), dtype=np.uint8).copy()
        self.running_comm_W = np.frombuffer(bytes(raw.running_comm_W), dtype=np.uint8).copy()
        self.running_comm_E = np.frombuffer(bytes(raw.running_comm_E), dtype=np.uint8).copy()
        self.ro_hash = np.frombuffer(bytes(raw.ro_hash), dtype=np.uint8).copy()
        self.status, self.seq = raw.status, raw.seq


class NovaFoldContext:
    def __init__(self, curve_id, ck_w, n_w, n_x, csr, depth=2, fmt=_capi.FMT_CANONICAL, ck_t=None, world=1, rank=0, latency_sms=0):
        """ck_w / ck_t: CommitmentKey (this rank's bases for W and for T/E; ck_t defaults to ck_w).
        csr: [(row_ptr u64, col u32, val bytes)] x 3 host arrays for A, B, C over z = (W, u, X)."""
        self.lib = _capi.lib()
        self.curve_id, self.n_w, self.n_x, self.depth = curve_id, n_w, n_x, depth
        self.n_rows = len(csr[0][0]) - 1
        self.world, self.rank = world, rank
        self._keep = [ck_w, ck_t]
        cfg = FoldConfig()
        cfg.curve_id, cfg.depth, cfg.n_w, cfg.n_x, cfg.n_rows = curve_id, depth, n_w, n_x, self.n_rows
        cfg.fmt, cfg.world, cfg.rank, cfg.latency_sms = fmt, world, rank, latency_sms
        arrs = []
        for m, (rp, col, val) in enumerate(csr):
            rp = np.ascontiguousarray(rp, dtype=np.uint64)
            col = np.ascontiguousarray(col, dtype=np.uint32)
            val = _u8(val)
            arrs += [rp, col, val]
            cfg.row_ptr[m] = rp.ctypes.data
            cfg.col[m] = col.ctypes.data if col.size else None
            cfg.val[m] = val.ctypes.data if val.size else None
        self._ctx = C.c_void_p()
        _capi.check(self.lib.lurk_fold_ctx_create(C.byref(cfg), ck_w._ctx, (ck_t or ck_w)._ctx, C.byref(self._ctx)))
        self.batches = []

    # ---- configuration
    def add_slot_batch(self, arity, offsets):
        """arity 0 = BitDecomp; offsets = element offset of every block inside W; returns the batch index"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        idx = self.lib.lurk_fold_ctx_add_slot_batch(self._ctx, arity, offs.size, offs.ctypes.data_as(C.c_void_p))
        if idx < 0:
            _capi.check(idx)
        self.batches.append((arity, offs.size))
        return idx

    def add_sha256_batch(self, n, offsets):
        """`len(offsets)` SHA-256 coprocessor calls with n pointers each (sha256.py); their witness blocks are written into W
        at these element offsets.  The batch's host buffer holds their inputs (per pointer tag, then hash); returns its index"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        idx = self.lib.lurk_fold_ctx_add_sha256_batch(self._ctx, n, offs.size, offs.ctypes.data_as(C.c_void_p))
        if idx < 0:
            _capi.check(idx)
        self.batches.append((("sha256", n), offs.size))
        return idx

    def add_trie_batch(self, op, height, offsets):
        """`len(offsets)` trie coprocessor calls (op trie.TRIE_LOOKUP / TRIE_INSERT at this height); their witness blocks
        are written into W at these element offsets.  The batch's host buffer holds their inputs (trie.lookup_inputs /
        insert_inputs), which stage A trusts: paths are not checked.  Returns its index"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        idx = self.lib.lurk_fold_ctx_add_trie_batch(self._ctx, op, height, offs.size, offs.ctypes.data_as(C.c_void_p))
        if idx < 0:
            _capi.check(idx)
        self.batches.append((("trie", op, height), offs.size))
        return idx

    def set_spans(self, spans):
        arr = (FoldSpan * len(spans))(*[FoldSpan(*map(int, s)) for s in spans])
        _capi.check(self.lib.lurk_fold_ctx_set_spans(self._ctx, len(spans), arr))

    def set_ro(self, kinds, challenge_bits=128):
        arr = (C.c_int * len(kinds))(*kinds)
        _capi.check(self.lib.lurk_fold_ctx_set_ro(self._ctx, len(kinds), arr, challenge_bits))

    def host_buffer(self, b, which):
        """numpy uint8 view of a pinned input buffer of fresh-instance buffer b (fill it, then stage_a(b))"""
        ptr, n = C.c_void_p(), C.c_size_t()
        _capi.check(self.lib.lurk_fold_ctx_host_buffer(self._ctx, b, which, C.byref(ptr), C.byref(n)))
        if not n.value:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(n.value,))

    def device_buffer(self, b, which):
        ptr, n = C.c_void_p(), C.c_size_t()
        _capi.check(self.lib.lurk_fold_ctx_device_buffer(self._ctx, b, which, C.byref(ptr), C.byref(n)))
        return ptr.value, n.value

    def read_device(self, b, which):
        """copy of a device buffer (tests): synchronises the context first"""
        self.sync()
        ptr, n = self.device_buffer(b, which)
        return device_tensor(ptr, n).cpu().numpy()

    def device_view(self, b, which):
        """torch view of a device buffer (e.g. to place device-resident inputs); order your writes against the context"""
        ptr, n = self.device_buffer(b, which)
        return device_tensor(ptr, n)

    # ---- multi-GPU: exchange buffers of the ranks (one process per GPU)
    def exchange_handle(self):
        h = np.zeros(64, dtype=np.uint8)
        _capi.check(self.lib.lurk_fold_ctx_exchange_handle(self._ctx, _capi.np_ptr(h)))
        return h

    def set_peers(self, handles):
        h = _u8(handles)
        assert h.size == 64 * self.world
        _capi.check(self.lib.lurk_fold_ctx_set_peers(self._ctx, _capi.np_ptr(h)))

    def connect(self, group=None):
        """all-gather the 64-byte exchange handles through torch.distributed and open the peers' buffers"""
        if self.world == 1:
            return
        import torch
        import torch.distributed as dist
        dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
        mine = torch.from_numpy(self.exchange_handle()).to(dev)
        allh = torch.empty(64 * self.world, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(allh, mine, group=group)
        self.set_peers(allh.cpu().numpy())

    # ---- running instance
    def set_running(self, W, E, u, X, comm_W, comm_E, fmt=_capi.FMT_CANONICAL):
        X = _u8(X) if self.n_x else np.zeros(32, dtype=np.uint8)
        _capi.check(self.lib.lurk_fold_ctx_set_running(self._ctx, _capi.np_ptr(_u8(W)), _capi.np_ptr(_u8(E)), _capi.np_ptr(_u8(u)), _capi.np_ptr(X),
                                                       _capi.np_ptr(_u8(comm_W)), _capi.np_ptr(_u8(comm_E)), fmt))

    def get_running(self, fmt=_capi.FMT_CANONICAL):
        W = np.zeros(self.n_w * 32, dtype=np.uint8)
        E = np.zeros(self.n_rows * 32, dtype=np.uint8)
        u = np.zeros(32, dtype=np.uint8)
        X = np.zeros(max(1, self.n_x) * 32, dtype=np.uint8)
        cw, ce = np.zeros(96, dtype=np.uint8), np.zeros(96, dtype=np.uint8)
        _capi.check(self.lib.lurk_fold_ctx_get_running(self._ctx, _capi.np_ptr(W), _capi.np_ptr(E), _capi.np_ptr(u), _capi.np_ptr(X), _capi.np_ptr(cw),
                                                       _capi.np_ptr(ce), fmt))
        return dict(W=W, E=E, u=u, X=X[:self.n_x * 32], comm_W=cw, comm_E=ce)

    # ---- steps
    def stage_a(self, b, resident=False, fmt=_capi.FMT_CANONICAL):
        _capi.check(self.lib.lurk_fold_ctx_stage_a(self._ctx, b, FOLD_INPUTS_RESIDENT if resident else 0, _capi.FMT_MONTGOMERY if resident else fmt))

    def init_running(self, b):
        _capi.check(self.lib.lurk_fold_ctx_init_running(self._ctx, b))

    def stage_b_launch(self, b):
        _capi.check(self.lib.lurk_fold_ctx_stage_b_launch(self._ctx, b))

    def collect(self, b, fmt=_capi.FMT_CANONICAL):
        raw = FoldResult()
        _capi.check(self.lib.lurk_fold_ctx_collect(self._ctx, b, C.byref(raw), fmt))
        return StepResult(raw)

    def check_running(self):
        """(rows violating the relaxed R1CS equation, comm_W consistent, comm_E consistent), computed on the device"""
        bad, okw, oke = C.c_uint64(), C.c_int(), C.c_int()
        _capi.check(self.lib.lurk_fold_ctx_check_running(self._ctx, C.byref(bad), C.byref(okw), C.byref(oke)))
        return bad.value, bool(okw.value), bool(oke.value)

    def stats(self):
        la, lb, aw, at = C.c_uint(), C.c_uint(), C.c_float(), C.c_float()
        _capi.check(self.lib.lurk_fold_ctx_stats(self._ctx, C.byref(la), C.byref(lb), C.byref(aw), C.byref(at)))
        return dict(launches_a=la.value, launches_b=lb.value, accumulate_w_ms=aw.value, accumulate_t_ms=at.value)

    def sync(self):
        _capi.check(self.lib.lurk_fold_ctx_sync(self._ctx))

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            self.lib.lurk_fold_ctx_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _DevView:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def device_tensor(ptr, n):
    """torch uint8 view of `n` bytes of device memory owned by the library (no copy)"""
    import torch
    return torch.as_tensor(_DevView(ptr, n), device="cuda")


class SuperNovaFoldContext:
    """NIVC (reference src/proof/supernova.rs:207-291): one running instance per circuit -- the Lurk step circuit plus one
    per coprocessor -- and every step folds into the instance selected by `MultiFrame::circuit_index()`
    (src/lem/multiframe.rs:941).  Each circuit has its own R1CS shape and buffers; they share the device-resident key."""

    def __init__(self, contexts):
        self.contexts = list(contexts)               # NovaFoldContext per circuit index
        self._next = [0] * len(self.contexts)        # next fresh-instance buffer per circuit
        self._started = [False] * len(self.contexts)

    def add_sha256_batch(self, circuit_index, n, offsets):
        """SHA-256 coprocessor calls of the circuit `circuit_index` (see NovaFoldContext.add_sha256_batch)"""
        return self.contexts[circuit_index].add_sha256_batch(n, offsets)

    def add_trie_batch(self, circuit_index, op, height, offsets):
        """trie coprocessor calls of the circuit `circuit_index` (see NovaFoldContext.add_trie_batch)"""
        return self.contexts[circuit_index].add_trie_batch(op, height, offsets)

    def stage_a(self, circuit_index, **kw):
        c = self.contexts[circuit_index]
        b = self._next[circuit_index]
        c.stage_a(b, **kw)
        self._next[circuit_index] = (b + 1) % c.depth
        return b

    def fold(self, circuit_index, b):
        """first step of a circuit initialises its running instance (RecursiveSNARK::new), later ones fold"""
        c = self.contexts[circuit_index]
        if not self._started[circuit_index]:
            c.init_running(b)
            self._started[circuit_index] = True
        else:
            c.stage_b_launch(b)

    def collect(self, circuit_index, b, **kw):
        return self.contexts[circuit_index].collect(b, **kw)
