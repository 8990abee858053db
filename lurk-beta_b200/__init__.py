"""lurk-beta_b200: H100 (sm_90a) implementation of lurk-beta's Nova/SuperNova proving hot path.

Only the path of SURVEY.md section 8: Poseidon digests and slot witnesses, store-DAG hydration, the Pedersen
commitment MSM and the fold helpers, behind the C ABI of include/lurk_b200.h (liblurk_b200.so).  This package is the
host-side mirror of the reference's interfaces for that path (PoseidonCache, StoreCore hydration, slot witnesses,
commitment key); it never computes on the CPU -- every call goes to the CUDA library and raises without it.
"""
from . import _capi, spartan
from ._capi import (CURVE_BN254_G1, CURVE_GRUMPKIN, CURVE_PALLAS, CURVE_VESTA, FIELD_BN254_FQ, FIELD_BN254_FR,
                    FIELD_PALLAS_FP, FIELD_PALLAS_FQ, FMT_CANONICAL, FMT_MONTGOMERY, LurkError)
from .commit import (CommitmentKey, ShardedCommitmentKey, ck_size, from_label, hash_to_curve_batch, point_sum, shake256, shard_bounds,
                     synthetic_bases)
from .fold import NovaFoldContext, SuperNovaFoldContext
from .hash import HashConstants, PoseidonCache
from .slots import SlotType, compute_witness_size, generate_slots_witnesses, slot_witness_batch_bytes
from .store import StoreCore
from .trie import StandardTrie, Trie

__all__ = [
    "CommitmentKey", "ShardedCommitmentKey", "NovaFoldContext", "SuperNovaFoldContext", "point_sum", "shard_bounds", "synthetic_bases", "ck_size", "from_label",
    "hash_to_curve_batch", "shake256", "spartan", "HashConstants", "PoseidonCache", "SlotType",
    "compute_witness_size", "generate_slots_witnesses", "slot_witness_batch_bytes", "StoreCore", "StandardTrie", "Trie", "LurkError",
    "FIELD_BN254_FR", "FIELD_BN254_FQ", "FIELD_PALLAS_FQ", "FIELD_PALLAS_FP", "CURVE_BN254_G1", "CURVE_GRUMPKIN",
    "CURVE_PALLAS", "CURVE_VESTA", "FMT_CANONICAL", "FMT_MONTGOMERY",
]
