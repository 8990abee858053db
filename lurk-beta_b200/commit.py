"""Pedersen commitments with a device-resident commitment key (reference: Arecibo CommitmentKey +
CommitmentEngineTrait::commit, reached from src/proof/nova.rs:287,292; key built in public_params,
src/proof/nova.rs:196-216).

`CommitmentKey` pins the whole key on the current GPU.  `ShardedCommitmentKey` is the N-GPU form: every rank owns a
contiguous slice of the bases, commits its slice of the scalars, and the ranks exchange the 96-byte partial points
with one all-gather (there is no NCCL reduction for elliptic-curve addition) and add them locally -- every rank gets
the same affine result.
"""
import ctypes as C

import numpy as np

from . import _capi


class CommitmentKey:
    def __init__(self, curve_id, bases, fmt=_capi.FMT_CANONICAL):
        """bases: uint8 array n*64 (affine x|y), host memory"""
        self.curve_id = curve_id
        bases = np.ascontiguousarray(bases, dtype=np.uint8).reshape(-1)
        if bases.size % 64:
            raise ValueError("bases buffer is not a whole number of affine points")
        self.n = bases.size // 64
        self._ctx = C.c_void_p()
        _capi.check(_capi.lib().lurk_msm_ctx_create(curve_id, _capi.np_ptr(bases), self.n, fmt, C.byref(self._ctx)))

    @classmethod
    def from_device(cls, curve_id, d_bases_ptr, n):
        """borrow bases already resident on the current device (Montgomery affine, n*64 bytes)"""
        self = cls.__new__(cls)
        self.curve_id, self.n = curve_id, n
        self._ctx = C.c_void_p()
        _capi.check(_capi.lib().lurk_msm_ctx_create_dev(curve_id, C.c_void_p(d_bases_ptr), n, C.byref(self._ctx)))
        return self

    @classmethod
    def setup(cls, curve_id, label, n, first=0):
        """Arecibo `CommitmentKey::setup(label, n)` = `DlogGroup::from_label` (public_params, src/proof/nova.rs:196-216): the
        key is generated on the GPU straight into the device buffer the commitment context reads (it never visits the host).
        first > 0: points first .. first + n - 1 of the key (a rank's slice of a sharded key)."""
        import torch
        buf = torch.empty(max(n, 1) * 64, dtype=torch.uint8, device="cuda")
        label = bytes(label)
        _capi.check(_capi.lib().lurk_ck_generate_range_dev(curve_id, label, len(label), first, n, C.c_void_p(buf.data_ptr()), None))
        self = cls.from_device(curve_id, buf.data_ptr(), n)
        self._bases = buf            # keeps the borrowed device memory alive
        return self

    @classmethod
    def powers_of_tau(cls, curve_id, g, beta, n):
        """the KZG engine's key (Arecibo hyperkzg CommitmentKey::setup -> gen_srs_for_testing): beta^i g for i < n, generated on the
        GPU into the buffer the context reads.  g: (x, y) ints, beta: int."""
        import torch
        buf = torch.empty(max(n, 1) * 64, dtype=torch.uint8, device="cuda")
        gb = np.frombuffer(int(g[0]).to_bytes(32, "little") + int(g[1]).to_bytes(32, "little"), dtype=np.uint8).copy()
        bb = np.frombuffer(int(beta).to_bytes(32, "little"), dtype=np.uint8).copy()
        _capi.check(_capi.lib().lurk_ck_powers_dev(curve_id, _capi.np_ptr(gb), _capi.np_ptr(bb), n, C.c_void_p(buf.data_ptr()), _capi.FMT_CANONICAL, None))
        self = cls.from_device(curve_id, buf.data_ptr(), n)
        self._bases = buf
        return self

    def commit(self, scalars, fmt=_capi.FMT_CANONICAL):
        """scalars: uint8 array n*32 (host) -> 96-byte point x|y|z (z = 1, or all zero for the identity)"""
        scalars = np.ascontiguousarray(scalars, dtype=np.uint8).reshape(-1)
        out = np.zeros(96, dtype=np.uint8)
        _capi.check(_capi.lib().lurk_msm_ctx_run(self._ctx, _capi.np_ptr(scalars), scalars.size // 32, fmt, _capi.np_ptr(out)))
        return out

    def commit_device(self, d_scalars_ptr, n, fmt=_capi.FMT_MONTGOMERY, stream=0):
        out = np.zeros(96, dtype=np.uint8)
        _capi.check(_capi.lib().lurk_msm_ctx_run_dev(self._ctx, C.c_void_p(d_scalars_ptr), n, fmt, _capi.np_ptr(out), C.c_void_p(stream)))
        return out

    def launch_device(self, d_scalars_ptr, n, fmt=_capi.FMT_MONTGOMERY, stream=0):
        """enqueue a commitment on `stream`; pair with finish()"""
        _capi.check(_capi.lib().lurk_msm_ctx_launch_dev(self._ctx, C.c_void_p(d_scalars_ptr), n, fmt, C.c_void_p(stream)))

    def finish(self):
        out = np.zeros(96, dtype=np.uint8)
        _capi.check(_capi.lib().lurk_msm_ctx_finish(self._ctx, _capi.np_ptr(out)))
        return out

    def precompute(self, window=0):
        """build the fixed-base window table on the device (once per key; call before clone()); window: width in bits instead of the
        one the key's size suggests (at 16 or less the digit sort keeps its histogram in shared memory)"""
        if window:
            _capi.check(_capi.lib().lurk_msm_ctx_precompute_window(self._ctx, window))
        else:
            _capi.check(_capi.lib().lurk_msm_ctx_precompute(self._ctx))
        return self

    def clone(self):
        """another context on the same device-resident key (own scratch), for overlapping commitments"""
        other = CommitmentKey.__new__(CommitmentKey)
        other.curve_id, other.n, other._parent = self.curve_id, self.n, self
        other._ctx = C.c_void_p()
        _capi.check(_capi.lib().lurk_msm_ctx_clone(self._ctx, C.byref(other._ctx)))
        return other

    def set_profiling(self, enable=True):
        _capi.check(_capi.lib().lurk_msm_ctx_set_profiling(self._ctx, 1 if enable else 0))

    def last_profile(self):
        """(device ms of the bucket-accumulation kernel, kernels launched) of the last run"""
        ms, k = C.c_float(), C.c_uint()
        _capi.check(_capi.lib().lurk_msm_ctx_last_profile(self._ctx, C.byref(ms), C.byref(k)))
        return ms.value, k.value

    def last_sort_ms(self):
        """device ms of the last run's digit sort (profiling enabled)"""
        ms = C.c_float()
        _capi.check(_capi.lib().lurk_msm_ctx_last_sort_ms(self._ctx, C.byref(ms)))
        return ms.value

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            _capi.lib().lurk_msm_ctx_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def synthetic_bases(curve_id, n, start=0, fmt=_capi.FMT_CANONICAL):
    """deterministic synthetic commitment key: [start+1]G .. [start+n]G, affine (host buffer, n*64 bytes)"""
    out = np.zeros(n * 64, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_synthetic_bases(curve_id, start, n, fmt, _capi.np_ptr(out)))
    return out


def ck_size(num_cons, num_vars, ck_floor=0):
    """R1CSShape::commitment_key: next_power_of_two(max(num_cons, num_vars, ck_floor)) bases"""
    return int(_capi.lib().lurk_ck_size(num_cons, num_vars, ck_floor))


def from_label(curve_id, label, n, fmt=_capi.FMT_CANONICAL):
    """DlogGroup::from_label(label, n) as a host buffer of n*64 bytes (affine x|y, identity = (0, 0))"""
    out = np.zeros(n * 64, dtype=np.uint8)
    label = bytes(label)
    _capi.check(_capi.lib().lurk_ck_generate(curve_id, label, len(label), n, fmt, _capi.np_ptr(out)))
    return out


def hash_to_curve_batch(curve_id, domain_prefix, messages, msg_len, fmt=_capi.FMT_CANONICAL):
    """Curve::hash_to_curve(domain_prefix)(m) for every msg_len-byte message of the buffer -> n*64 bytes"""
    messages = np.ascontiguousarray(messages, dtype=np.uint8).reshape(-1)
    n = messages.size // msg_len if msg_len else 0
    out = np.zeros(n * 64, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_hash_to_curve_batch(curve_id, domain_prefix.encode(), _capi.np_ptr(messages), msg_len, n, fmt,
                                                     _capi.np_ptr(out)))
    return out


def shake256(data, out_len):
    """host-side SHAKE256 of the library (the XOF behind from_label)"""
    data = bytes(data)
    out = np.zeros(out_len, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_shake256(data, len(data), _capi.np_ptr(out), out_len))
    return out.tobytes()


def point_sum(curve_id, points, fmt=_capi.FMT_CANONICAL):
    """sum of 96-byte result points on the host (the combine step of the sharded commit)"""
    points = np.ascontiguousarray(points, dtype=np.uint8).reshape(-1)
    out = np.zeros(96, dtype=np.uint8)
    _capi.check(_capi.lib().lurk_point_sum(curve_id, _capi.np_ptr(points), points.size // 96, fmt, _capi.np_ptr(out)))
    return out


def shard_bounds(n, world_size, rank):
    """contiguous slice [lo, hi) of an n-element key owned by `rank`"""
    per = (n + world_size - 1) // world_size
    lo = min(n, rank * per)
    return lo, min(n, lo + per)


class ShardedCommitmentKey:
    """Commitment key sharded over the ranks of a torch.distributed process group (one process per GPU)."""

    def __init__(self, curve_id, local_bases, n_total, group=None, fmt=_capi.FMT_CANONICAL):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.curve_id = curve_id
        self.n_total = n_total
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.lo, self.hi = shard_bounds(n_total, self.world, self.rank)
        self.local = CommitmentKey(curve_id, local_bases, fmt)
        assert self.local.n == self.hi - self.lo

    def combine(self, partial, fmt=_capi.FMT_CANONICAL):
        """all-gather the 96-byte partial points and add them (identical result on every rank)"""
        import torch
        dev = "cuda" if self.dist.get_backend(self.group) == "nccl" else "cpu"
        mine = torch.from_numpy(np.ascontiguousarray(partial, dtype=np.uint8)).to(dev)
        gathered = torch.empty(96 * self.world, dtype=torch.uint8, device=dev)
        self.dist.all_gather_into_tensor(gathered, mine, group=self.group)
        return point_sum(self.curve_id, gathered.cpu().numpy(), fmt)

    def commit_local(self, local_scalars, fmt=_capi.FMT_CANONICAL):
        return self.local.commit(local_scalars, fmt)

    def commit(self, local_scalars, fmt=_capi.FMT_CANONICAL):
        """local_scalars: this rank's slice [lo, hi) of the scalar vector"""
        return self.combine(self.commit_local(local_scalars, fmt), fmt)
