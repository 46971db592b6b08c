"""icicle_b200: H100 (sm_90a) MSM + NTT + vec-ops engine behind ICICLE's device-backend API.

The package holds only what the hot path needs: csrc/ (CUDA kernels + the C ABI of include/icicle_b200.h), shim/ (the
C++ registration shims that plug the C ABI into ICICLE's REGISTER_*_BACKEND hooks) and this thin Python mirror of the
reference frontend used by tests/ and bench.py.  Importing it requires the built native library (no fallback).
"""
from .api import *  # noqa: F401,F403
from .api import Field, Curve, NTTDir, Ordering, MSMConfig, NTTConfig, VecOpsConfig, MatMulConfig, HashConfig, Poseidon2, MerkleTreeConfig, MerkleTree, PaddingPolicy, HashKind, Hasher, PowConfig, proof_of_work, proof_of_work_verify, IcicleError  # noqa: F401
from . import utils  # noqa: F401

__version__ = "0.1.0"
