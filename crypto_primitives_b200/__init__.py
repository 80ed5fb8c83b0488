"""crypto_primitives_b200 -- H100-native (sm_90a CUDA) batched evaluation of the
ark-crypto-primitives hot path: Poseidon CRH / two-to-one, Pedersen CRH / commitment, and the
Merkle-tree build over them, behind the reference's CRHScheme / TwoToOneCRHScheme /
CommitmentScheme / merkle_tree::Config surface.  All hashing happens in libcpb200.so
(csrc/, C-ABI in include/cpb200.h); this package is the host-side mirror of the reference's
interface plus ctypes plumbing.  There is no CPU fallback: importing fails without the library,
and every compute call fails without an H100.
"""
from . import _native
from .fields import BLS12_381_FR, BLS12_377_FR, BN254_FR, ED_ON_BLS12_377_FR, JUBJUB_FR, FIELDS, Field
from .sponge.poseidon import (PoseidonConfig, PoseidonSponge, PoseidonSpongeBatch, RaggedPoseidonSpongeBatch, absorb_squeeze_batch, absorb_squeeze_ragged, find_poseidon_ark_and_mds,
                              get_default_poseidon_parameters)
from .crh import poseidon as crh_poseidon
from .crh import pedersen as crh_pedersen
from .crh import bowe_hopwood as crh_bowe_hopwood
from .commitment import pedersen as commitment_pedersen
from .commitment import blake2s as commitment_blake2s
from .signature import schnorr as signature_schnorr
from .signature.schnorr import Schnorr
from .encryption import elgamal as encryption_elgamal
from .encryption.elgamal import ElGamal
from . import curves
from . import merkle_tree

__all__ = ["Field", "FIELDS", "BLS12_381_FR", "BN254_FR", "JUBJUB_FR", "BLS12_377_FR", "ED_ON_BLS12_377_FR", "PoseidonConfig", "PoseidonSponge", "PoseidonSpongeBatch", "RaggedPoseidonSpongeBatch", "absorb_squeeze_batch",
           "absorb_squeeze_ragged",
           "find_poseidon_ark_and_mds", "get_default_poseidon_parameters", "crh_poseidon", "crh_pedersen", "crh_bowe_hopwood", "commitment_pedersen",
           "commitment_blake2s", "signature_schnorr", "Schnorr", "encryption_elgamal", "ElGamal", "curves", "merkle_tree"]
