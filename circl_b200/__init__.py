"""circl_b200 -- H100 (sm_90a) batch polynomial-ring engine for CIRCL's
module-lattice hot path (ML-KEM / ML-DSA).

The product is ``libcirclb200.so`` (hand-written CUDA behind the C ABI in
``include/circl_b200.h``).  The Python modules here are a thin host-side mirror
of the reference's interfaces used by the tests and the bench:

  circl_b200.kyber   -- pke/kyber/internal/common Poly method surface (batched)
  circl_b200.mlkem   -- kem.Scheme for ML-KEM-768 / ML-KEM-1024 (+ batch methods)
  circl_b200.keccak  -- simd/keccakf1600 + internal/sha3 (batched permutation and one-shot sponges)
"""
from ._ffi import Cb200Error, lib, check  # noqa: F401
from .runtime import (host_batch, host_free, init, init_devices, active_devices, bind_thread_to_device, release_stream, shutdown,  # noqa: F401
                      device_count, set_stream, synchronize, launch_count)
