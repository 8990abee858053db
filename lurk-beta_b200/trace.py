"""Reader / writer of the reference-side trace files (SURVEY.md 8(f) N1).

A lurk-beta built with `--features b200-trace` (integration/rust/trace_export.patch, applied to
src/lem/multiframe.rs:520-592) writes one `slots_<step>.bin` per call of `generate_slots_witnesses`: every slot's aux
assignment exactly as Neptune's circuit2 / bellpepper's `to_bits_le_strict` allocated it.  These files are the only thing
that can PIN the aux order of lurk_poseidon_witness_batch / lurk_bitdecomp_witness_batch (the reference pins sizes only,
src/lem/multiframe.rs:991-1016); tests/test_trace_fixtures.py checks every file found under tests/golden/traces/.
`commit_<n>.bin` (an Arecibo-side dump of one `commit` call: key slice, scalars, result; INTEGRATION.md section 5) pins the
byte encoding of commitments the same way.

All integers little-endian; field elements 32 bytes canonical (`PrimeField::to_repr`).
  slots file : "LRKS" | u32 version=1 | u32 field (0 BN256, 1 Grumpkin, 2 Pallas, 3 Vesta) | u32 flags (bit 0: synthetic,
               written by this module, not by the reference) | u32 n_slots |
               n_slots x { u8 slot_type (0 Hash4, 1 Hash6, 2 Hash8, 3 Commitment, 4 BitDecomp) | u8 is_dummy | u16 0 |
                           u32 len | len x 32 bytes }
  commit file: "LRKC" | u32 version=1 | u32 curve (0 BN254 G1, 1 Grumpkin, 2 Pallas, 3 Vesta) | u32 flags | u32 n |
               n x 64 bytes affine bases (x | y; identity = 0 | 0) | n x 32 bytes scalars | 64 bytes affine result | u8 is_identity
  sha256 file: "LRKH" | u32 version=1 | u32 field | u32 flags | u32 n | 2n x 32 bytes inputs (tag, hash per pointer) |
               u32 len | len x 32 bytes aux -- one call of the SHA-256 coprocessor's `synthesize_sha256`
               (src/coprocessor/sha256.rs:27-64) and the aux block it allocated: pins the aux order of
               lurk_sha256_witness_batch (tests/test_trace_sha256.py).
  trie file  : "LRKT" | u32 version=1 | u32 field | u32 flags | u32 op (0 lookup, 1 insert) | u32 height | u32 n_in |
               n_in x 32 bytes inputs | u32 len | len x 32 bytes aux -- one call of the trie coprocessor's
               synthesize_lookup_aux / synthesize_insert_aux (src/coprocessor/trie/mod.rs:118-156, 226-268), its inputs as
               lurk_trie_witness_batch takes them and the aux block it allocated (tests/test_trace_trie.py).
  key file   : "LRKK" | u32 version=1 | u32 curve | u32 flags | u32 kind (0 = from_label / Pedersen, 1 = powers of tau / KZG) |
               u32 label_len | label | u32 n | n x 64 bytes affine points -- the head of the reference's commitment key as
               `CommitmentKey::setup(label, ..)` produced it (SURVEY.md 8(f) N3): pins lurk_ck_generate (kind 0).  For kind 1 the label
               field holds g (64 bytes) | beta (32 bytes) as the reference's seeded RNG drew them: pins lurk_ck_powers_dev.
"""
import struct
from collections import namedtuple

import numpy as np

SLOT_TYPES = ("Hash4", "Hash6", "Hash8", "Commitment", "BitDecomp")
SLOT_ARITY = {"Hash4": 4, "Hash6": 6, "Hash8": 8, "Commitment": 3, "BitDecomp": 0}
FLAG_SYNTHETIC = 1
# LanguageField order of the exporter -> field ids of include/lurk_b200.h
TRACE_FIELD_TO_ID = {0: 0, 1: 1, 2: 2, 3: 3}

Slot = namedtuple("Slot", "slot_type is_dummy witness")          # witness: uint8 array, len * 32 bytes
SlotTrace = namedtuple("SlotTrace", "field_id synthetic slots")
CommitTrace = namedtuple("CommitTrace", "curve_id synthetic bases scalars result is_identity")
Sha256Trace = namedtuple("Sha256Trace", "field_id synthetic n inputs aux")   # inputs: 2n * 32 bytes, aux: len * 32 bytes
TrieTrace = namedtuple("TrieTrace", "field_id synthetic op height inputs aux")   # inputs: n_in * 32 bytes, aux: len * 32
KeyTrace = namedtuple("KeyTrace", "curve_id synthetic kind label points")     # points: uint8 array, n * 64 bytes


def write_slots(path, field_id, slots, synthetic=True):
    out = [b"LRKS", struct.pack("<IIII", 1, field_id, FLAG_SYNTHETIC if synthetic else 0, len(slots))]
    for s in slots:
        w = np.ascontiguousarray(s.witness, dtype=np.uint8).reshape(-1)
        assert w.size % 32 == 0
        out.append(struct.pack("<BBHI", SLOT_TYPES.index(s.slot_type), 1 if s.is_dummy else 0, 0, w.size // 32))
        out.append(w.tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(out))


def read_slots(path):
    data = open(path, "rb").read()
    if data[:4] != b"LRKS":
        raise ValueError(f"{path}: not a slot trace")
    version, field, flags, n = struct.unpack_from("<IIII", data, 4)
    if version != 1:
        raise ValueError(f"{path}: unknown version {version}")
    off, slots = 20, []
    for _ in range(n):
        typ, dummy, _pad, ln = struct.unpack_from("<BBHI", data, off)
        off += 8
        slots.append(Slot(SLOT_TYPES[typ], bool(dummy), np.frombuffer(data, dtype=np.uint8, count=ln * 32, offset=off).copy()))
        off += ln * 32
    if off != len(data):
        raise ValueError(f"{path}: trailing bytes")
    return SlotTrace(TRACE_FIELD_TO_ID[field], bool(flags & FLAG_SYNTHETIC), slots)


def write_commit(path, curve_id, bases, scalars, result_affine, is_identity, synthetic=True):
    bases = np.ascontiguousarray(bases, dtype=np.uint8).reshape(-1)
    scalars = np.ascontiguousarray(scalars, dtype=np.uint8).reshape(-1)
    n = scalars.size // 32
    assert bases.size == 64 * n
    with open(path, "wb") as f:
        f.write(b"LRKC" + struct.pack("<IIII", 1, curve_id, FLAG_SYNTHETIC if synthetic else 0, n))
        f.write(bases.tobytes() + scalars.tobytes() + np.ascontiguousarray(result_affine, dtype=np.uint8).reshape(-1)[:64].tobytes())
        f.write(bytes([1 if is_identity else 0]))


def read_commit(path):
    data = open(path, "rb").read()
    if data[:4] != b"LRKC":
        raise ValueError(f"{path}: not a commitment trace")
    version, curve, flags, n = struct.unpack_from("<IIII", data, 4)
    if version != 1:
        raise ValueError(f"{path}: unknown version {version}")
    off = 20
    bases = np.frombuffer(data, dtype=np.uint8, count=64 * n, offset=off).copy()
    off += 64 * n
    scalars = np.frombuffer(data, dtype=np.uint8, count=32 * n, offset=off).copy()
    off += 32 * n
    result = np.frombuffer(data, dtype=np.uint8, count=64, offset=off).copy()
    ident = bool(data[off + 64])
    if off + 65 != len(data):
        raise ValueError(f"{path}: trailing bytes")
    return CommitTrace(curve, bool(flags & FLAG_SYNTHETIC), bases, scalars, result, ident)


def write_sha256(path, field_id, n, inputs, aux, synthetic=True):
    inputs = np.ascontiguousarray(inputs, dtype=np.uint8).reshape(-1)
    aux = np.ascontiguousarray(aux, dtype=np.uint8).reshape(-1)
    assert inputs.size == 64 * n and aux.size % 32 == 0
    with open(path, "wb") as f:
        f.write(b"LRKH" + struct.pack("<IIII", 1, field_id, FLAG_SYNTHETIC if synthetic else 0, n) + inputs.tobytes())
        f.write(struct.pack("<I", aux.size // 32) + aux.tobytes())


def read_sha256(path):
    data = open(path, "rb").read()
    if data[:4] != b"LRKH":
        raise ValueError(f"{path}: not a SHA-256 trace")
    version, field, flags, n = struct.unpack_from("<IIII", data, 4)
    if version != 1 or n < 1:
        raise ValueError(f"{path}: unknown version / empty call")
    off = 20
    inputs = np.frombuffer(data, dtype=np.uint8, count=64 * n, offset=off).copy()
    off += 64 * n
    (ln,) = struct.unpack_from("<I", data, off)
    off += 4
    aux = np.frombuffer(data, dtype=np.uint8, count=32 * ln, offset=off).copy()
    if off + 32 * ln != len(data):
        raise ValueError(f"{path}: trailing bytes")
    return Sha256Trace(TRACE_FIELD_TO_ID[field], bool(flags & FLAG_SYNTHETIC), n, inputs, aux)


def write_trie(path, field_id, op, height, inputs, aux, synthetic=True):
    inputs = np.ascontiguousarray(inputs, dtype=np.uint8).reshape(-1)
    aux = np.ascontiguousarray(aux, dtype=np.uint8).reshape(-1)
    assert inputs.size % 32 == 0 and aux.size % 32 == 0
    with open(path, "wb") as f:
        f.write(b"LRKT" + struct.pack("<IIIIII", 1, field_id, FLAG_SYNTHETIC if synthetic else 0, op, height, inputs.size // 32))
        f.write(inputs.tobytes() + struct.pack("<I", aux.size // 32) + aux.tobytes())


def read_trie(path):
    data = open(path, "rb").read()
    if data[:4] != b"LRKT":
        raise ValueError(f"{path}: not a trie trace")
    version, field, flags, op, height, n_in = struct.unpack_from("<IIIIII", data, 4)
    if version != 1 or op not in (0, 1) or height < 1:
        raise ValueError(f"{path}: unknown version / op / height")
    off = 28
    inputs = np.frombuffer(data, dtype=np.uint8, count=32 * n_in, offset=off).copy()
    off += 32 * n_in
    (ln,) = struct.unpack_from("<I", data, off)
    off += 4
    aux = np.frombuffer(data, dtype=np.uint8, count=32 * ln, offset=off).copy()
    if off + 32 * ln != len(data):
        raise ValueError(f"{path}: trailing bytes")
    return TrieTrace(TRACE_FIELD_TO_ID[field], bool(flags & FLAG_SYNTHETIC), op, height, inputs, aux)


def write_key(path, curve_id, kind, label, points, synthetic=True):
    points = np.ascontiguousarray(points, dtype=np.uint8).reshape(-1)
    assert points.size % 64 == 0
    label = bytes(label)
    with open(path, "wb") as f:
        f.write(b"LRKK" + struct.pack("<IIIII", 1, curve_id, FLAG_SYNTHETIC if synthetic else 0, kind, len(label)) + label)
        f.write(struct.pack("<I", points.size // 64) + points.tobytes())


def read_key(path):
    data = open(path, "rb").read()
    if data[:4] != b"LRKK":
        raise ValueError(f"{path}: not a commitment-key trace")
    version, curve, flags, kind, ll = struct.unpack_from("<IIIII", data, 4)
    if version != 1 or kind not in (0, 1):
        raise ValueError(f"{path}: unknown version / kind")
    off = 24
    label = data[off:off + ll]
    off += ll
    (n,) = struct.unpack_from("<I", data, off)
    off += 4
    pts = np.frombuffer(data, dtype=np.uint8, count=64 * n, offset=off).copy()
    if off + 64 * n != len(data):
        raise ValueError(f"{path}: trailing bytes")
    return KeyTrace(curve, bool(flags & FLAG_SYNTHETIC), kind, label, pts)


def slot_batches(trace):
    """group the slots of a trace per slot type, in file order: {slot_type: (preimages uint8, witnesses uint8, indices)}.
    The preimage of a slot is the head of its witness block (allocate_slot allocates it first, src/lem/circuit.rs:264-299)."""
    out = {}
    for i, s in enumerate(trace.slots):
        a = SLOT_ARITY[s.slot_type] or 1
        out.setdefault(s.slot_type, ([], [], []))
        pre, wit, idx = out[s.slot_type]
        pre.append(s.witness[:a * 32])
        wit.append(s.witness)
        idx.append(i)
    return {k: (np.concatenate(p), np.concatenate(w), i) for k, (p, w, i) in out.items()}
