"""The C-ABI library loads and exports every symbol include/cpb200.h declares; host-only entry
points (parameter generation, argument validation) behave like the reference.  No GPU needed."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import ROOT, kats
import crypto_primitives_b200 as cp
from crypto_primitives_b200 import _native as N
from oracle import fields as OF


def test_every_declared_symbol_is_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "cpb200.h")).read()
    declared = set(re.findall(r"\b(cpb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = C.CDLL(N.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in cpb200.h but not exported"
    assert declared == set(N.SIGNATURES), declared ^ set(N.SIGNATURES)
    assert N.lib.cpb_abi_version() == int(re.search(r"#define CPB_ABI_VERSION (\d+)", hdr).group(1))
    # the status codes of the header and of the ctypes binding agree
    status_enum = hdr[hdr.index("typedef enum cpb_status"):hdr.index("} cpb_status;")]
    codes = dict(re.findall(r"(CPB_[A-Z0-9_]+) = (\d+)", status_enum))
    assert len(codes) == 10
    for name, value in codes.items():
        assert getattr(N, name) == int(value), name


def test_moduli():
    for f in cp.FIELDS.values():
        assert f.modulus == OF.MODULI[f.name]


def test_default_parameters_match_reference_kats():
    K = kats()["default_params"]
    f = cp.BLS12_381_FR
    for weights in (False, True):
        for rate in range(2, 9):
            cfg = cp.get_default_poseidon_parameters(f, rate, weights)
            e = K["weights" if weights else "constraints"][str(rate)]
            assert f.to_ints(cfg.ark[0, 0])[0] == int(e["ark00"])
            assert f.to_ints(cfg.mds[0, 0])[0] == int(e["mds00"])
            assert cfg.capacity == 1 and cfg.rate == rate
    assert cp.get_default_poseidon_parameters(f, 9, False) is None          # traits.rs:102 -> None
    assert cp.get_default_poseidon_parameters(f, 1, False) is None
    # the tables belong to BLS12-381 Fr (R/sponge/test.rs:13-32); no other field has an impl in the reference
    for other in (cp.BN254_FR, cp.JUBJUB_FR, cp.BLS12_377_FR):
        assert cp.get_default_poseidon_parameters(other, 2, False) is None
        assert cp.get_default_poseidon_parameters(other, 3, True) is None


def test_find_ark_and_mds_rejects_wrong_bit_size():
    a = np.zeros((39, 3, 4), dtype=np.uint64)
    m = np.zeros((3, 3, 4), dtype=np.uint64)
    st = N.lib.cpb_poseidon_find_ark_and_mds(0, 254, 2, 8, 31, 0, a.ctypes.data_as(N.u64p), m.ctypes.data_as(N.u64p))
    assert st == N.CPB_BAD_PARAMS and b"MODULUS_BIT_SIZE" in N.lib.cpb_last_error()


def test_ctx_create_validates_before_touching_the_gpu():
    out = N.vp()
    a = np.zeros((39, 3, 4), dtype=np.uint64)
    m = np.zeros((3, 3, 4), dtype=np.uint64)
    assert N.lib.cpb_poseidon_ctx_create(9, 2, 1, 8, 31, 17, a.ctypes.data_as(N.u64p), m.ctypes.data_as(N.u64p), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    assert N.lib.cpb_poseidon_ctx_create(0, 0, 1, 8, 31, 17, a.ctypes.data_as(N.u64p), m.ctypes.data_as(N.u64p), 0, C.byref(out)) == N.CPB_BAD_PARAMS
    bad = a.copy()
    bad[0, 0] = np.uint64(0xFFFFFFFFFFFFFFFF)                               # not reduced
    assert N.lib.cpb_poseidon_ctx_create(0, 2, 1, 8, 31, 17, bad.ctypes.data_as(N.u64p), m.ctypes.data_as(N.u64p), 0, C.byref(out)) == N.CPB_BAD_PARAMS


@pytest.mark.skipif(N.lib.cpb_device_count() > 0, reason="an H100 is present")
def test_no_cpu_fallback_without_device():
    """Without a GPU the compute path must fail loudly, never fall back."""
    cfg = cp.get_default_poseidon_parameters(cp.BLS12_381_FR, 2, False)
    with pytest.raises(N.CpbError) as e:
        cp.crh_poseidon.CRH.evaluate(cfg, cp.BLS12_381_FR.elements([0, 1, 2]))
    assert e.value.status in (N.CPB_NO_DEVICE, N.CPB_CUDA_ERROR)


def test_absorb_encodings_host_side():
    """sponge/absorb.py is pure host logic (R/sponge/absorb.rs): checked here against the oracle's restatement without a GPU
    (only cpb_field_modulus, a host function of the library, is called)."""
    import crypto_primitives_b200 as cp
    from crypto_primitives_b200.sponge import absorb as A
    from oracle import absorb as OA
    f = cp.BLS12_381_FR
    p = f.modulus
    pairs = [([1, -2, 3], [1, -2, 3]), (bytes(range(64)), bytes(range(64))), ("str", "str"), (None, None), (False, False),
             (A.Some(A.usize(5)), OA.Some(OA.UInt(5, 64))), (A.WithLength(b"abc"), OA.WithLength(b"abc")),
             (A.Elems(f, f.elements([5, p - 1])), [OA.Fe(5, p), OA.Fe(p - 1, p)]), (A.UInt(2**127, 128), OA.UInt(2**127, 128)),
             (A.Point(cp.curves.JUBJUB, f.elements([3, 4])), OA.TEPoint(3, 4, p))]
    for g, o in pairs:
        assert A.to_sponge_bytes(g) == OA.to_sponge_bytes(o)
        assert f.to_ints(A.to_sponge_field_elements(g, f)) == OA.to_sponge_field_elements(o, p)


def test_generic_config_level_loop_heap_order():
    """merkle_tree.Config's generic build (used by configs without a fused device build, e.g. Bowe-Hopwood trees) fills the
    reference's heap-ordered arrays (R/merkle_tree/mod.rs:446-523); checked with a toy hash on the host."""
    import numpy as np
    from crypto_primitives_b200.merkle_tree import Config

    class Toy(Config):
        def leaf_hash_batch(self, prm, leaves, device):
            return (np.asarray(leaves, dtype=np.uint64) * np.uint64(3) + np.uint64(1)).reshape(-1, 4)

        def two_to_one_batch(self, prm, pairs, device):
            p = np.asarray(pairs, dtype=np.uint64)
            return p[:, 0] * np.uint64(5) + p[:, 1] * np.uint64(7) + np.uint64(11)

    n = 16
    leaves = np.arange(n * 4, dtype=np.uint64).reshape(n, 4)
    ln, nn = Toy().build(None, None, leaves, 0)
    assert ln.shape == (n, 4) and nn.shape == (n - 1, 4)
    full = np.concatenate([nn, ln])
    for i in range(n - 1):
        assert np.array_equal(full[i], full[2 * i + 1] * np.uint64(5) + full[2 * i + 2] * np.uint64(7) + np.uint64(11))
    import pytest
    with pytest.raises(ValueError):
        Toy().build_from_digests(None, ln[:6], 0)


def test_multi_gpu_entry_points_validate_their_arguments():
    """cpb_exchange_* / cpb_multi_* reject bad shapes before touching a device (include/cpb200.h, "Merkle tree across
    several GPUs"); CPB_NCCL_ERROR is part of the status enum a shim must map."""
    h = N.vp()
    for world, rank in ((3, 0), (0, 0), (4, 4), (2, -1), (32, 0)):
        assert N.lib.cpb_exchange_create(0, world, rank, C.byref(h)) == N.CPB_BAD_PARAMS
    devs = (C.c_int * 3)(0, 1, 2)
    assert N.lib.cpb_multi_create(3, devs, C.byref(h)) == N.CPB_BAD_PARAMS           # not a power of two
    dup = (C.c_int * 2)(0, 0)
    assert N.lib.cpb_multi_create(2, dup, C.byref(h)) == N.CPB_BAD_PARAMS            # the same device twice
    assert N.lib.cpb_multi_create(2, None, C.byref(h)) == N.CPB_NULL_POINTER
    assert N.lib.cpb_merkle_poseidon_build_multi(None, None, None, None, 2, 4, None, None) == N.CPB_NULL_POINTER
    assert N.lib.cpb_exchange_world(None) == 0 and N.lib.cpb_exchange_rank(None) == -1 and N.lib.cpb_multi_uses_nccl(None) == 0
    assert N.CPB_NCCL_ERROR == 9
    assert N.lib.cpb_host_register(None, 16) == N.CPB_NULL_POINTER
