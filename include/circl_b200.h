/*
 * include/circl_b200.h -- C ABI of libcirclb200.so, the H100 (sm_90a) batch
 * polynomial-ring engine behind CIRCL's module-lattice hot path.
 *
 * This is the surface a cgo shim binds (see INTEGRATION.md and go/).  Plain
 * pointers and sizes only.  Every buffer is caller-owned and never retained
 * past the call.  A pointer may be a host pointer (pageable or pinned) or a
 * CUDA device pointer; the library detects which (cudaPointerGetAttributes)
 * and stages host buffers through HBM itself.  All entry points return 0 on
 * success or a negative code; cb200_last_error() gives the message.  There is
 * no CPU fallback: without a usable CUDA device every compute call fails.
 *
 * Citations are file:line in cloudflare/circl (the interface each entry point
 * replaces).  Coefficient order is the reference's standard ("detangled")
 * order; results are bit-identical to the reference's *Generic functions.
 */
#ifndef CIRCL_B200_H
#define CIRCL_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes (mapped by the Go shim to kem.Err*, kem/kem.go:92-121) ---- */
#define CB200_OK 0
#define CB200_ERR_ARG (-1)          /* programmer error: the Go shim panics, as the reference does */
#define CB200_ERR_NOT_INIT (-2)
#define CB200_ERR_PUBKEY (-3)       /* kem.ErrPubKey: ek not reduced mod q (cpapke.go:45-55); see cb200_mlkem_encaps */
#define CB200_ERR_SIGN_ATTEMPTS (-4)/* ML-DSA: 576 attempts exhausted (sign/mldsa/mldsa65/internal/dilithium.go:372-377) */
#define CB200_ERR_PRIVKEY (-5)      /* kem.ErrPrivKey: H(ek) inside dk does not match (kem/mlkem/mlkem768/kyber.go:226-228) */
/* <= -100: CUDA runtime error (-100 - cudaError_t) */

/* ---- lifetime ---- */
/* cb200_init_devices(ndev): one process drives GPUs 0..ndev-1 (ndev <= 0: every visible GPU).  Host-pointer batch
 * calls are then cut into one contiguous index range per GPU inside the library and the results land in the
 * caller's buffers in index order -- a kem.Scheme / sign.Scheme caller never sees devices (north_star: "batches
 * shard by index across the 8 GPUs").  cb200_init(device): exactly one GPU (the one-process-per-GPU launch).
 * Calling either again with another set re-initialises. */
int cb200_init(int device);
int cb200_init_devices(int ndev);
int cb200_active_devices(void);        /* GPUs this process was initialised on (0 = not initialised) */
void cb200_shutdown(void);
int cb200_device_count(void);
const char *cb200_last_error(void);    /* message of the last failing call on this thread */
const char *cb200_version(void);
/* Threading (kem/kem.go:33-82 and sign/sign.go:48-94 are goroutine-safe; so is this):
 *  - host-pointer calls may be issued from any number of threads; each GPU runs the ranges it is given one after
 *    the other on its own worker thread, small batches rotate over the GPUs;
 *  - device-pointer calls run on the GPU that owns the buffers, asynchronously on the CUDA stream (cudaStream_t cast
 *    to void*) the CALLING THREAD named with cb200_set_stream -- the setting is per thread; NULL, the initial state,
 *    is CUDA's legacy default stream.  Scratch memory is kept per (GPU, stream): calls on different streams never
 *    share it, calls on one stream from several threads are serialised in stream order.  cb200_release_stream frees
 *    the scratch of a stream that is about to be destroyed.  A cgo caller wraps set_stream + call in
 *    runtime.LockOSThread (go/cb200). */
int cb200_set_stream(void *cuda_stream);
int cb200_release_stream(void *cuda_stream);
int cb200_synchronize(void);           /* waits for this thread's stream */
/* Pins the calling thread to the CPUs next to GPU `device` (/sys/bus/pci/devices/<id>/local_cpulist); memory it
 * allocates and first touches afterwards is local to that GPU's NUMA node.  Returns the number of CPUs, 0 if the
 * topology is unknown (affinity unchanged).  The library's own worker threads do this themselves. */
int cb200_bind_thread_to_device(int device);
/* ---- result gather of the one-process-per-GPU launch (SURVEY.md 8(e)) ----
 * Rank 0 allocates the destination of the gather (plain cudaMalloc memory on its GPU) and gets a 64-byte handle to
 * publish over any transport (torch.distributed, a pipe); every other rank opens the handle and pushes its rows:
 * cb200_gather_push(dst, src, bytes) is a cudaMemcpyAsync into the mapped peer memory over NVLink, issued on a copy
 * stream of the library that first waits for everything the calling thread's stream has queued so far -- copy-engine
 * traffic, no SM, no NCCL kernel beside the compute kernels.  dst may also be local (rank 0's own rows).
 * cb200_gather_flush(row, wait_on_host): wait_on_host != 0 blocks until this rank's pushes have landed; otherwise the
 * calling thread's stream is made to wait for them.  `row` is any device pointer of the pushing GPU. */
#define CB200_GATHER_HANDLE_BYTES 64
int cb200_gather_alloc(size_t bytes, void **dev_ptr, uint8_t *handle);
int cb200_gather_free(void *dev_ptr);
int cb200_gather_open(const uint8_t *handle, void **peer_ptr);
int cb200_gather_close(void *peer_ptr);
int cb200_gather_push(void *dst, const void *src, size_t bytes);
int cb200_gather_flush(const void *any_local_row, int wait_on_host);
/* Pinned host memory for large batches handed to Go via unsafe.Slice. */
void *cb200_host_alloc(size_t bytes);
/* The same for one array of a batch (n rows of unit_bytes) that host-pointer calls will split over all active GPUs
 * (cb200_init_devices): the rows of each GPU's shard are placed on that GPU's NUMA node, so that all GPUs copy at link
 * speed at the same time instead of sharing the socket interconnect.  Freed with cb200_host_free. */
void *cb200_host_alloc_batch(size_t n, size_t unit_bytes);
void cb200_host_free(void *p);
/* number of kernels launched by this library since init (bench accounting) */
uint64_t cb200_launch_count(void);
/* Optional per-kernel-class timing with CUDA events on the launching stream
 * (used by bench.py for the roofline line).  cb200_profile_read synchronises the
 * device, fills ms_total[i] / launches[i] for the first n classes and clears. */
int cb200_profile_enable(int on);
int cb200_profile_kernel_count(void);
const char *cb200_profile_kernel_name(int id);
int cb200_profile_read(double *ms_total, uint64_t *launches, int n);

/* ---- Kyber / ML-KEM ring, q = 3329, Poly = [256]int16 ---- */
/* (*Poly).NTT / InvNTT   pke/kyber/internal/common/generic.go:24,36; stubs_amd64.go:8-14
 * in place over n contiguous polynomials.  Results equal nttGeneric / invNTTGeneric (ntt.go:60-193) bit for bit,
 * unnormalised, for EVERY int16 input (the reference's int16 wrap-around included).  Inputs inside the reference's
 * contract (|c| <= q; in fact |c| <= 13561 forward, <= 3679 inverse) run a faster kernel path. */
int cb200_kyber_ntt(int16_t *polys, size_t n, int inverse);
/* (*Poly).MulHat         generic.go:49; poly.go:63-100.  out may alias a or b. */
int cb200_kyber_mulhat(int16_t *out, const int16_t *a, const int16_t *b, size_t n);
/* PolyDotHat             pke/kyber/kyber768/internal/vec.go:30-37
 * a, b: n vectors of k polynomials; out: n polynomials. */
int cb200_kyber_dot(int16_t *out, const int16_t *a, const int16_t *b, int k, size_t n);
/* Add, Sub, BarrettReduce, Normalize, ToMont   generic.go:7-77, poly.go:13-52 */
#define CB200_OP_ADD 0
#define CB200_OP_SUB 1
#define CB200_OP_BARRETT 2
#define CB200_OP_NORMALIZE 3
#define CB200_OP_TOMONT 4
int cb200_kyber_poly_op(int op, int16_t *out, const int16_t *a, const int16_t *b, size_t n);

/* ---- Dilithium / ML-DSA ring, q = 8380417, Poly = [256]uint32 ---- */
/* (*Poly).NTT / InvNTT   sign/internal/dilithium/generic.go:11,15; stubs_amd64.go:8-14; in place */
int cb200_dil_ntt(uint32_t *polys, size_t n, int inverse);
/* (*Poly).MulHat         sign/internal/dilithium/generic.go:19 (poly.go:88) */
int cb200_dil_mulhat(uint32_t *out, const uint32_t *a, const uint32_t *b, size_t n);
/* PolyDotHat             sign/mldsa/mldsa65/internal/mat.go:52-59 (k = L polynomials per vector) */
int cb200_dil_dot(uint32_t *out, const uint32_t *a, const uint32_t *b, int k, size_t n);
/* Add, Sub, ReduceLe2Q, Normalize, NormalizeAssumingLe2Q, MulBy2toD   generic.go:23-89, poly.go:10-100 */
#define CB200_DIL_OP_ADD 0
#define CB200_DIL_OP_SUB 1
#define CB200_DIL_OP_REDUCE_LE2Q 2
#define CB200_DIL_OP_NORMALIZE 3
#define CB200_DIL_OP_NORMALIZE_LE2Q 4
#define CB200_DIL_OP_MUL_2D 5
int cb200_dil_poly_op(int op, uint32_t *out, const uint32_t *a, const uint32_t *b, size_t n);
/* (*Poly).Exceeds        poly.go:51-71 (stubs_amd64.go:32 exceedsAVX2): flags[i] = 1 iff poly i exceeds bound */
int cb200_dil_exceeds(const uint32_t *polys, uint32_t bound, uint8_t *flags, size_t n);

/* ---- Keccak (simd/keccakf1600, internal/sha3): the on-device sampler's permutation, batched ---- */
/* StateX4.Permute  simd/keccakf1600/f1600x.go:115-121 / KeccakF1600  internal/sha3/keccakf.go:12
 * states: n x 25 little-endian 64-bit lanes (200 bytes per state, lane x+5y at index x+5y), permuted in place;
 * turbo != 0: the 12-round TurboSHAKE variant (keccakf.go:12 `turbo`). */
int cb200_keccak_f1600(uint64_t *states, size_t n, int turbo);
/* One-shot sponges over n messages of equal length (internal/sha3/hashes.go:21,35; shake.go:56,74):
 * bits = 128 / 256 selects SHAKE128 / SHAKE256 with `outlen` output bytes, bits = -256 / -512 selects SHA3-256 /
 * SHA3-512 (outlen must be 32 / 64).  Message i = in + i*in_stride (in_stride 0: one message), output i at
 * out + i*outlen. */
int cb200_sha3(int bits, const uint8_t *in, size_t in_stride, size_t inlen, uint8_t *out, size_t outlen, size_t n);

/* ---- samplers of the Kyber ring (pke/kyber/internal/common/sample.go) ---- */
/* (*Poly).DeriveUniform  sample.go:192-236: polys[i] = 12-bit rejection sampling of SHAKE128(seed_i || x_i || y_i);
 * seeds: 32 bytes each at seeds + i*seed_stride (0: one seed); xy: n x 2 bytes (x, y). */
int cb200_kyber_derive_uniform(int16_t *polys, const uint8_t *seeds, size_t seed_stride, const uint8_t *xy, size_t n);
/* (*Poly).DeriveNoise(2|3)  sample.go:31-95: polys[i] = CBD_eta(SHAKE256(seed_i || nonce_i)); seeds 32 bytes each. */
int cb200_kyber_derive_noise(int16_t *polys, int eta, const uint8_t *seeds, size_t seed_stride, const uint8_t *nonces,
                             size_t n);
/* ---- serialisation of the Kyber ring (pke/kyber/internal/common/poly.go) ---- */
/* Pack / Unpack  poly.go:106-129: 12 bits per coefficient, 384 bytes per polynomial (input normalised) */
int cb200_kyber_pack(uint8_t *out, const int16_t *polys, size_t n);
int cb200_kyber_unpack(int16_t *polys, const uint8_t *in, size_t n);
/* CompressTo / Decompress  poly.go:170-328 for d in {4, 5, 10, 11} (32 d bytes per polynomial), and
 * CompressMessageTo / DecompressMessage  poly.go:134-166 for d = 1 (32 bytes); compress expects normalised input */
int cb200_kyber_compress(uint8_t *out, const int16_t *polys, int d, size_t n);
int cb200_kyber_decompress(int16_t *polys, const uint8_t *in, int d, size_t n);

/* ---- samplers and packers of the Dilithium ring; mode = 44, 65 or 87 picks the per-mode package
 *      (sign/mldsa/mldsa{44,65,87}/internal/sample.go, sign/internal/dilithium/generic.go) ---- */
/* PolyDeriveUniform  sample.go:92-123: 23-bit rejection sampling of SHAKE128(seed_i || le16(nonce_i)); seeds 32 bytes */
int cb200_dil_derive_uniform(uint32_t *polys, const uint8_t *seeds, size_t seed_stride, const uint16_t *nonces, size_t n);
/* PolyDeriveUniformLeqEta  sample.go:129-181: coefficients Q + eta - t, t from nibbles of SHAKE256(seed_i(64) || nonce) */
int cb200_dil_derive_leq_eta(int mode, uint32_t *polys, const uint8_t *seeds, size_t seed_stride, const uint16_t *nonces,
                             size_t n);
/* PolyDeriveUniformLeGamma1  sample.go:197-209: gamma1 - (18|20-bit fields of SHAKE256(seed_i(64) || nonce)), mod q */
int cb200_dil_derive_le_gamma1(int mode, uint32_t *polys, const uint8_t *seeds, size_t seed_stride,
                               const uint16_t *nonces, size_t n);
/* PolyDeriveUniformBall  sample.go:299-339: tau coefficients +-1 from SHAKE256(seed_i); seeds are c~ (32/48/64 bytes
 * for mode 44/65/87) at seeds + i*seed_stride */
int cb200_dil_derive_ball(int mode, uint32_t *polys, const uint8_t *seeds, size_t seed_stride, size_t n);
/* (*Poly).Power2Round  generic.go:85 (poly.go:77-84): a0plusq[i] = Q + a0, a1[i] for normalised a */
int cb200_dil_power2round(uint32_t *a0plusq, uint32_t *a1, const uint32_t *a, size_t n);
/* (*Poly).PackLe16  generic.go:27 (pack.go:102-108): 4 bits per coefficient, 128 bytes per polynomial */
int cb200_dil_pack_le16(uint8_t *out, const uint32_t *polys, size_t n);

/* ---- ML-KEM ---- */
/* scheme.UnmarshalBinaryPublicKey + EncapsulateDeterministically
 *   kem/mlkem/mlkem768/kyber.go:390-396,359-374,103-137 (mlkem1024: same lines)
 * k = 2 (ML-KEM-512: ek 800, ct 768), 3 (ML-KEM-768: ek 1184, ct 1088) or 4 (ML-KEM-1024: ek 1568, ct 1568).
 * ek_stride = 0: one ek shared by all n operations (parsed once);
 * otherwise op i uses ek + i*ek_stride and A^T, H(ek) are rebuilt on device per op.
 * seeds: n x 32 (the message m); ct: n x CiphertextSize; ss: n x 32.
 * status (optional, may be NULL): n bytes, 0 = ok, 1 = kem.ErrPubKey for that op
 * (its ct/ss are zeroed).  Returns CB200_ERR_PUBKEY if any op failed. */
int cb200_mlkem_encaps(int k, const uint8_t *ek, size_t ek_stride, const uint8_t *seeds, uint8_t *ct, uint8_t *ss,
                       uint8_t *status, size_t n);
/* The same on device pointers, with the result gather of the one-process-per-GPU launch fused into the flow: the rows of
 * every sub-batch (4096 operations) are also copied to push_ct + i*CiphertextSize / push_ss + i*32 -- typically this
 * rank's place in rank 0's cb200_gather_alloc buffer, opened with cb200_gather_open -- as soon as they exist, by the
 * copy engines over NVLink while the following sub-batches compute.  Either may be NULL.  The calling thread's stream
 * is ordered after the pushes. */
int cb200_mlkem_encaps_push(int k, const uint8_t *ek, size_t ek_stride, const uint8_t *seeds, uint8_t *ct, uint8_t *ss,
                            uint8_t *status, size_t n, uint8_t *push_ct, uint8_t *push_ss);
/* scheme.UnmarshalBinaryPrivateKey + Decapsulate
 *   kem/mlkem/mlkem768/kyber.go:398-407,376-388 -> PrivateKey.Unpack :203-229, DecapsulateTo :144-184
 *   (cpapke DecryptTo cpapke.go:113-130, re-encryption EncryptTo :137-181, implicit rejection with J = SHAKE256(z || ct)).
 * dk: packed decapsulation key(s) (2400 / 3168 bytes); op i uses dk + i*dk_stride (0 = one key, host pointers only).
 * ct: n x CiphertextSize; ss: n x 32.  status (optional): 2 = kem.ErrPrivKey for that op (ss zeroed).
 * Returns CB200_ERR_PRIVKEY if any op failed. */
int cb200_mlkem_decaps(int k, const uint8_t *dk, size_t dk_stride, const uint8_t *ct, uint8_t *ss, uint8_t *status,
                       size_t n);
/* scheme.DeriveKeyPair   kem/mlkem/mlkem768/kyber.go:337-346 -> NewKeyFromSeed :57-78 ->
 *   cpapke.NewKeyFromSeedMLKEM pke/kyber/kyber768/kyber.go:77-86 -> internal/cpapke.go:66-110.
 * seeds: n x 64 (d || z); ek: n x PublicKeySize; dk: n x PrivateKeySize (packed, = MarshalBinary). */
int cb200_mlkem_keygen(int k, const uint8_t *seeds, uint8_t *ek, uint8_t *dk, size_t n);
size_t cb200_mlkem_private_key_size(int k);
size_t cb200_mlkem_public_key_size(int k);
size_t cb200_mlkem_ciphertext_size(int k);

#define CB200_SIGN_INTERNAL 1 /* flags: ML-DSA.Sign_internal / Verify_internal on the message as given */

/* ---- round-3 Kyber512/768/1024 KEM (k = 2, 3, 4): kem/kyber/kyber768/kyber.go:56-198 ----
 * Same K-PKE and byte sizes as ML-KEM; the FO wrapper differs (m = H(seed), ss = KDF(K || H(ct)), key generation
 * without the K byte, no modulus check of ek, no H(ek) check of dk -- hence no status array).  Strides as in
 * cb200_mlkem_*: 0 = one key shared by all operations. */
int cb200_kyber_kem_keygen(int k, const uint8_t *seeds, uint8_t *ek, uint8_t *dk, size_t n);
int cb200_kyber_kem_encaps(int k, const uint8_t *ek, size_t ek_stride, const uint8_t *seeds, uint8_t *ct, uint8_t *ss,
                           size_t n);
int cb200_kyber_kem_decaps(int k, const uint8_t *dk, size_t dk_stride, const uint8_t *ct, uint8_t *ss, size_t n);

/* ---- callers on the wire side of ML-KEM (SURVEY.md 8(f) row 4) ----
 * cb200_x25519: dh/x25519 KeyGen (points == NULL: base point, key.go:44-46) or Shared (key.go:48-56) on n
 * 32-byte scalars / points; status[i] = 1 where the point has small order (Shared returning false); the output is
 * then all zero and the host-pointer call returns CB200_ERR_PUBKEY after finishing the batch. */
int cb200_x25519(const uint8_t *scalars, const uint8_t *points, uint8_t *out, uint8_t *status, size_t n);
/* dh/x448 KeyGen (points == NULL: u = 5, key.go:33-35) or Shared (key.go:41-46) on n 56-byte scalars / points;
 * status and return value as cb200_x25519 (low order: the residue mod p is 0, 1 or p - 1, curve.go:76-104).
 * Device pointers: 8-byte aligned. */
int cb200_x448(const uint8_t *scalars, const uint8_t *points, uint8_t *out, uint8_t *status, size_t n);

/* X-Wing (kem/xwing/xwing.go:32-44): seed / sk 32, pk 1216 (ML-KEM-768 ek || X25519 pk), encapsulation seed 64,
 * ct 1120, ss 32.  keygen = DeriveKeyPairPacked (:131-141; the packed sk is the seed itself), encaps = Encapsulate
 * (:173-182, kem.ErrPubKey through status / CB200_ERR_PUBKEY as in cb200_mlkem_encaps), decaps = Decapsulate
 * (:185-191, which re-derives the key pair from the 32-byte sk). */
int cb200_xwing_keygen(const uint8_t *seeds, uint8_t *pk, size_t n);
int cb200_xwing_encaps(const uint8_t *pk, size_t pk_stride, const uint8_t *eseeds, uint8_t *ct, uint8_t *ss,
                       uint8_t *status, size_t n);
int cb200_xwing_decaps(const uint8_t *sk, size_t sk_stride, const uint8_t *ct, uint8_t *ss, size_t n);

/* kem/hybrid (hybrid.go:197-283 over xkem.go): keys, ciphertexts and shared secrets are the two halves side by side
 * in the order of hybrid.go:34-93.  The sizes follow from the id (cb200_hybrid_*_size): shared secret 64 for the
 * X25519 hybrids and 88 for the X448 ones, key seed 64, encapsulation seed 32 (X25519) or 56 (X448).
 * status bit 0 = kem.ErrPubKey (non-canonical ML-KEM ek or low-order X25519 / X448 share), bit 1 = kem.ErrPrivKey.
 * Device pointers and strides: 16-byte aligned for ids 0-2, 8-byte aligned for ids 3-4. */
#define CB200_HYBRID_X25519MLKEM768 0  /* ML-KEM-768 || X25519:  pk 1216, sk 2432, ct 1120 */
#define CB200_HYBRID_KYBER768_X25519 1 /* X25519 || Kyber768:    pk 1216, sk 2432, ct 1120 */
#define CB200_HYBRID_KYBER512_X25519 2 /* X25519 || Kyber512:    pk 832,  sk 1664, ct 800  */
#define CB200_HYBRID_KYBER768_X448  3  /* X448 || Kyber768:      pk 1240, sk 2456, ct 1144, ss 88 */
#define CB200_HYBRID_KYBER1024_X448 4  /* X448 || Kyber1024:     pk 1624, sk 3224, ct 1624, ss 88 */
int cb200_hybrid_keygen(int id, const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_hybrid_encaps(int id, const uint8_t *pk, size_t pk_stride, const uint8_t *seeds, uint8_t *ct, uint8_t *ss,
                        uint8_t *status, size_t n);
int cb200_hybrid_decaps(int id, const uint8_t *sk, size_t sk_stride, const uint8_t *ct, uint8_t *ss, uint8_t *status,
                        size_t n);
size_t cb200_hybrid_public_key_size(int id);
size_t cb200_hybrid_private_key_size(int id);
size_t cb200_hybrid_ciphertext_size(int id);
size_t cb200_hybrid_shared_key_size(int id);         /* 64 for ids 0-2, 88 for ids 3-4 */
size_t cb200_hybrid_seed_size(int id);               /* 64 for every id */
size_t cb200_hybrid_encapsulation_seed_size(int id); /* 32 for ids 0-2, 56 for ids 3-4 */

/* ---- HPKE DHKEMs (RFC 9180 section 4.1; hpke/kembase.go, hpke/xkem.go), as kem/schemes registers them ----
 * The ids are the HPKE KEM identifiers.  X25519: seed, encapsulation seed, pk, sk and enc 32 bytes, ss 32 (HKDF-SHA256);
 * X448: all 56 bytes, ss 64 (HKDF-SHA512).
 * keygen = DeriveKeyPair (xkem.go:55-71): sk = LabeledExpand(LabeledExtract("", "dkp_prk", seed), "sk", "", Nsk),
 *   stored unclamped; pk = KeyGen(sk).
 * encaps = Encap with DeriveKeyPair(seed) as the ephemeral key (kembase.go:120-183); decaps = Decap (:185-241), which
 *   recomputes pkR from skR.  auth_encaps / auth_decaps = AuthEncap / AuthDecap (:133-159,194-217) with the sender's
 *   skS / pkS.  kem_context holds the key and enc bytes exactly as passed (X25519: bit 255 included).
 * Strides: 0 = one key for the whole batch (its public key is then computed once per call).
 * status: status[i] = 1 where a DH step met a low-order point (x25519/x448.Shared returning false); that op's ss is
 *   all zero.  A host-pointer call finishes the batch and returns CB200_ERR_PUBKEY (the reference's
 *   hpke.ErrInvalidKEMSharedSecret); a device-pointer call reports only through status, which it requires.
 * An unknown id is CB200_ERR_ARG.  Device pointers and strides: 16-byte aligned for 0x20, 8-byte aligned for 0x21. */
#define CB200_HPKE_X25519_HKDF_SHA256 0x20
#define CB200_HPKE_X448_HKDF_SHA512 0x21
int cb200_hpke_keygen(int id, const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_hpke_encaps(int id, const uint8_t *pkR, size_t pkR_stride, const uint8_t *seeds, uint8_t *enc, uint8_t *ss,
                      uint8_t *status, size_t n);
int cb200_hpke_decaps(int id, const uint8_t *skR, size_t skR_stride, const uint8_t *enc, uint8_t *ss, uint8_t *status,
                      size_t n);
int cb200_hpke_auth_encaps(int id, const uint8_t *pkR, size_t pkR_stride, const uint8_t *skS, size_t skS_stride,
                           const uint8_t *seeds, uint8_t *enc, uint8_t *ss, uint8_t *status, size_t n);
int cb200_hpke_auth_decaps(int id, const uint8_t *skR, size_t skR_stride, const uint8_t *enc, const uint8_t *pkS,
                           size_t pkS_stride, uint8_t *ss, uint8_t *status, size_t n);
size_t cb200_hpke_public_key_size(int id);
size_t cb200_hpke_private_key_size(int id);
size_t cb200_hpke_ciphertext_size(int id);
size_t cb200_hpke_shared_key_size(int id);
size_t cb200_hpke_seed_size(int id);
size_t cb200_hpke_encapsulation_seed_size(int id);

/* ---- P-256 ECDH (Go's crypto/ecdh.P256(), as the reference's hpke/shortkem.go uses it) ----
 * cb200_p256: KeyGen (points == NULL: out = 0x04 || X || Y of [k]G, 65-byte rows) or Shared (out = X of [k]P, 32-byte
 * rows) on n 32-byte big-endian scalars and 65-byte uncompressed points.  A scalar must satisfy 0 < k < n
 * (ecdh.NewPrivateKey), a point must be 0x04 || X || Y with X, Y < p on the curve (ecdh.NewPublicKey).
 * status (optional): bit 0 = invalid point, bit 1 = invalid scalar; a failed op's output row is all zero.  A
 * host-pointer call finishes the batch and returns CB200_ERR_PRIVKEY if any scalar failed, else CB200_ERR_PUBKEY if any
 * point failed.  Device pointers may start at any byte. */
int cb200_p256(const uint8_t *scalars, const uint8_t *points, uint8_t *out, uint8_t *status, size_t n);

/* ---- HPKE DHKEM(P-256, HKDF-SHA256), kem_id 0x10 (hpke/shortkem.go, hpke/kembase.go; hpke/algs.go:248-253) ----
 * The cb200_hpke_* contracts above without the id; the generic entry points keep treating 0x10 as unknown.
 * Sizes: seed, encapsulation seed and sk 32 (a big-endian scalar), pk and enc 65 (0x04 || X || Y), ss 32.
 * keygen = DeriveKeyPair (shortkem.go:63-90): the first candidate LabeledExpand(dkp_prk, "candidate", I2OSP(ctr, 1), 32),
 *   ctr = 0..255, that lies in [1, n - 1].
 * kem_context is enc || pkR (130 bytes) or enc || pkR || pkS (195); the auth dh is dh1 || dh2 (64).
 * status bit 0 = hpke.ErrInvalidKEMPublicKey (pkR, enc or pkS is not a P-256 point), bit 1 =
 *   hpke.ErrInvalidKEMPrivateKey (skR or skS is not in [1, n - 1]); that op's ss is all zero and its enc is still
 *   written.  A key shared by the batch (stride 0) that fails marks every op.  A host-pointer call finishes the batch,
 *   then returns CB200_ERR_PRIVKEY if any op has bit 1, else CB200_ERR_PUBKEY if any has bit 0; a device-pointer call
 *   reports only through status, which it requires.
 * Strides: 0 = one key for the whole batch.  65-byte rows cannot all be aligned, so device pointers and strides may
 * start at any byte. */
#define CB200_HPKE_P256_HKDF_SHA256 0x10
int cb200_hpke_p256_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_hpke_p256_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *seeds, uint8_t *enc, uint8_t *ss,
                           uint8_t *status, size_t n);
int cb200_hpke_p256_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, uint8_t *ss, uint8_t *status,
                           size_t n);
int cb200_hpke_p256_auth_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *skS, size_t skS_stride,
                                const uint8_t *seeds, uint8_t *enc, uint8_t *ss, uint8_t *status, size_t n);
int cb200_hpke_p256_auth_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, const uint8_t *pkS,
                                size_t pkS_stride, uint8_t *ss, uint8_t *status, size_t n);
size_t cb200_hpke_p256_public_key_size(void);             /* 65 */
size_t cb200_hpke_p256_private_key_size(void);            /* 32 */
size_t cb200_hpke_p256_ciphertext_size(void);             /* 65 */
size_t cb200_hpke_p256_shared_key_size(void);             /* 32 */
size_t cb200_hpke_p256_seed_size(void);                   /* 32 */
size_t cb200_hpke_p256_encapsulation_seed_size(void);     /* 32 */

/* ---- OPRF servers (RFC 9497) over the NIST curves: the reference's oprf package (oprf/oprf.go, server.go, keys.go,
 * zk/dleq/dleq.go:84-243, group/short.go:100-135,246-283,404-470, expander/expander.go) ----
 * suite: one of the ids below (the suite ids of the CFRG drafts); mode: 0 (Server), 1 (VerifiableServer) or 2
 * (PartialObliviousServer).  Elements are compressed points (0x02 | 0x03 || X, Ne bytes), scalars Ns big-endian bytes.
 * An unknown suite or mode, an info longer than 65535 bytes (oprf.ErrInvalidInfo) or a null required pointer is
 * CB200_ERR_ARG.  Key rows have a stride (0 = one key for the batch).  Rows of device buffers may start at any byte.
 * status (required, one byte per op, all-zero outputs on failure): 1 = a blinded element does not decode
 * (group.UnmarshalBinary), 2 = sk not in [1, n - 1] (oprf.ErrInvalidPrivateKey), 4 = r not in [1, n - 1], 8 = mode 2
 * with t = sk + HashToScalar(info) = 0 (oprf.ErrInverseZero), 16 = a FullEvaluate input over 65535 bytes on a
 * device-pointer call.  The call itself returns 0. */
#define CB200_OPRF_P256_SHA256 3 /* Ne 33, Ns 32, Nh 32, proof 64 */
#define CB200_OPRF_P384_SHA384 4 /* Ne 49, Ns 48, Nh 48, proof 96 */
#define CB200_OPRF_P521_SHA512 5 /* Ne 67, Ns 66, Nh 64, proof 132 */
size_t cb200_oprf_element_size(int suite); /* Ne; 0 for an unknown suite */
size_t cb200_oprf_scalar_size(int suite);  /* Ns */
size_t cb200_oprf_output_size(int suite);  /* Nh */
size_t cb200_oprf_proof_size(int suite);   /* 2 Ns: c || s */
/* DeriveKey (keys.go:103-132): 32-byte seeds, one info for the batch -> sk (Ns) and pk = compress([sk]G) (Ne). */
int cb200_oprf_derive_key(int suite, int mode, const uint8_t *seeds, const uint8_t *info, size_t info_len, uint8_t *sk,
                          uint8_t *pk, size_t n);
/* Evaluate (server.go:23-85): n requests of m blinded elements each (1 <= m <= 65535, n * m rows of Ne) -> evaluated
 * (n * m rows of Ne) and, in modes 1 and 2, one proof per request (2 Ns) from the randomness rnd (one Ns row per
 * request, the reference's rand.Reader draw; rnd and proof are ignored in mode 0).  info: mode 2 only. */
int cb200_oprf_evaluate(int suite, int mode, const uint8_t *sk, size_t sk_stride, const uint8_t *blinded, size_t m,
                        const uint8_t *rnd, const uint8_t *info, size_t info_len, uint8_t *evaluated, uint8_t *proof,
                        uint8_t *status, size_t n);
/* FullEvaluate (server.go:97-117): input i is msgs[msg_off[i] .. msg_off[i + 1]) -> out (Nh).  Inputs are limited to
 * 65535 bytes as RFC 9497 bounds them (the reference silently truncates the length prefix instead): a host-pointer
 * call refuses a longer one with CB200_ERR_ARG before any device work; on a device-pointer call, whose offsets the
 * host does not read, that op gets status bit 16 and an all-zero output.  info: mode 2 only.
 * VerifyFinalize is this call followed by a constant-time compare. */
int cb200_oprf_full_evaluate(int suite, int mode, const uint8_t *sk, size_t sk_stride, const uint8_t *msgs,
                             const uint64_t *msg_off, const uint8_t *info, size_t info_len, uint8_t *out,
                             uint8_t *status, size_t n);

/* ---- RSA blind signatures (RFC 9474, RSABSSA-SHA384), server side: the reference's blindsign/blindrsa package
 * (brsa.go:202-257, internal/common/common.go:80-93,121-137, internal/common/pss.go:132-221) ----
 * variant: the reference's Variant order below.  Keys are big-endian byte strings (leading zero bytes allowed), one
 * key per call, always in host memory: N of 2048 to 4096 bits and an odd e with 3 <= e < 2^32 (and, for BlindSign, two
 * primes of at most 2048 bits each).  Anything else, a null
 * required pointer or an unknown variant is CB200_ERR_ARG with a message, before the device is touched.  Rows are
 * kLen = ceil(bitlen(N) / 8) bytes (cb200_brsa_modulus_bytes) and on device buffers may start at any byte.  The status
 * bytes are required; a failed op's output row is all zero and the call itself returns 0. */
#define CB200_BRSA_SHA384_PSS_RANDOMIZED 0         /* salt 48 bytes, 32-byte message prefix */
#define CB200_BRSA_SHA384_PSSZERO_RANDOMIZED 1     /* salt 0 */
#define CB200_BRSA_SHA384_PSS_DETERMINISTIC 2      /* salt 48, no prefix */
#define CB200_BRSA_SHA384_PSSZERO_DETERMINISTIC 3  /* salt 0 */
size_t cb200_brsa_modulus_bytes(const uint8_t *N, size_t N_len); /* kLen; 0 outside 2048 to 4096 bits */
/* Signer.BlindSign (brsa.go:237-257): blinded (n rows of kLen) -> sig = c^d mod N (n rows of kLen), from the PKCS #1
 * CRT fields (the two primes with p q = N, dp = d mod (p - 1), dq = d mod (q - 1), qinv = q^-1 mod p, each at most as
 * many 32-bit words as the larger prime).  The exponentiation is constant-time in place of the reference's base
 * blinding, so the call takes no randomness.  status: 1 = c > N (ErrInvalidMessageLength), 2 = s^e mod N != c
 * (DecryptAndCheck's "rsa: internal error", also the result of c = N or of inconsistent CRT fields). */
int cb200_brsa_blind_sign(const uint8_t *N, size_t N_len, const uint8_t *e, size_t e_len, const uint8_t *p,
                          size_t p_len, const uint8_t *q, size_t q_len, const uint8_t *dp, size_t dp_len,
                          const uint8_t *dq, size_t dq_len, const uint8_t *qinv, size_t qinv_len,
                          const uint8_t *blinded, uint8_t *sig, uint8_t *status, size_t n);
/* Verifier.Verify (brsa.go:214): message i = msgs[msg_off[i] .. msg_off[i + 1]) (n + 1 offsets; for the randomized
 * variants the prepared message, prefix included) and sigs (n rows of kLen).  status: 0 = valid, 1 = s >= N,
 * 2 = an inconsistent EMSA-PSS encoding (both rsa.ErrVerification in the reference).  Messages are limited to
 * 2^31 - 1 bytes: a host-pointer call refuses offsets that decrease or a longer message with CB200_ERR_ARG before any
 * device work; on a device-pointer call, whose offsets the host does not read, that op gets status 2. */
int cb200_brsa_verify(int variant, const uint8_t *N, size_t N_len, const uint8_t *e, size_t e_len,
                      const uint8_t *msgs, const uint64_t *msg_off, const uint8_t *sigs, uint8_t *status, size_t n);

/* ---- Partially blind RSA signatures (draft-amjad-cfrg-partially-blind-rsa, RSAPBSSA-SHA384), server side: the
 * reference's blindsign/blindrsa/partiallyblindrsa package (pbrsa.go) ----
 * Each op's metadata selects the key: e' from HKDF-SHA-384 of the metadata (derivePublicKey, pbrsa.go:81-117) and
 * d' = e'^-1 mod phi(N).  Keys follow the cb200_brsa_* rules (big-endian byte strings in host memory, one key per
 * call, N of 2048 to 4096 bits, primes of at most 2048 bits with p q = N); in addition p and q must be = 3 mod 4 and
 * qinv = q^-1 mod p below p.  Metadata i is meta[meta_off[i] .. meta_off[i + 1]) (n + 1 offsets), at most 2^31 - 8
 * bytes, and in Verify metadata and message together are at most 2^31 - 8 bytes.  A host-pointer call refuses offsets
 * that decrease or longer strings with CB200_ERR_ARG, like any other argument error, before the device is touched; on a
 * device-pointer call, whose offsets the host does not read, that op gets status 2.  Rows are kLen bytes
 * (cb200_brsa_modulus_bytes) and on device buffers may start at any byte.  The status bytes are required; a failed
 * op's output row is all zero and the call itself returns 0. */
/* NewSigner's safe-prime test (pbrsa.go:324-343): 20 Miller-Rabin rounds with random bases on (p - 1) / 2 and
 * (q - 1) / 2, on the host (no device needed).  0, or CB200_ERR_ARG with a message.  BlindSign does not repeat it: a key
 * that passes by chance fails every op with status 2. */
int cb200_pbrsa_check_key(const uint8_t *N, size_t N_len, const uint8_t *p, size_t p_len, const uint8_t *q,
                          size_t q_len);

/* ---- Prio3 aggregators (draft-irtf-cfrg-vdaf-14): the reference's vdaf/prio3 package, aggregator side ----
 * One instance is a cb200_prio3_config: kind (the reference's algorithm ID, which the XOF header also hashes), the
 * number of shares (2..255), the circuit's parameters (only those of its kind are read: Sum max_measurement; SumVec
 * length, bits, chunk_length; Histogram length, chunk_length; MultiHotCountVec length, max_weight, chunk_length) and
 * the application context (at most 65527 bytes, host memory).  A configuration the reference's New refuses
 * (ErrNumShares, ErrContextSize, the circuits' parameter errors), an unknown kind, an agg_id >= num_shares (ErrAggID),
 * a null required pointer, or a circuit whose PrepInit work area exceeds 64 MiB per report (about 2^22 Field128
 * elements: measurement, proof and a 2^k-point Lagrange domain) is CB200_ERR_ARG before the device is touched.
 * Every row is the reference's wire encoding (elements little-endian, 8 bytes in Field64 for Count and Sum, 16 in
 * Field128 for the others; seeds 32 bytes; nonces 16 bytes); cb200_prio3_get_sizes gives the lengths.  Rows are dense, one
 * per report, and device rows may start at any byte.  Buffers are all host or all device memory.
 * status (required, one byte per report): 1 = an element that does not decode (a leader input-share element or a
 * prep-share element >= p, UnmarshalBinary), 2 = ErrJointRand (PrepInit: the report's joint-rand part does not match
 * the public share; PrepNext: the prep message's seed is not the corrected one), 4 = ErrInvalidEval (t^p = 1), 8 =
 * ErrProofVerify (Decide rejects).  The outputs of a failed report are all zero; the call itself returns 0. */
#define CB200_PRIO3_COUNT 1
#define CB200_PRIO3_SUM 2
#define CB200_PRIO3_SUMVEC 3
#define CB200_PRIO3_HISTOGRAM 4
#define CB200_PRIO3_MULTIHOT 5
typedef struct {
  uint32_t kind;
  uint32_t num_shares;
  uint64_t max_measurement; /* Sum */
  uint64_t length;          /* SumVec, Histogram, MultiHotCountVec */
  uint64_t bits;            /* SumVec */
  uint64_t chunk_length;    /* SumVec, Histogram, MultiHotCountVec */
  uint64_t max_weight;      /* MultiHotCountVec */
  const uint8_t *context;
  size_t context_len;
} cb200_prio3_config;
typedef struct {
  size_t input_share_leader; /* meas share || proof share (|| blind) */
  size_t input_share_helper; /* seed (|| blind) */
  size_t public_share;       /* num_shares joint-rand parts, or 0 */
  size_t prep_share;         /* verifier share (|| joint-rand part) */
  size_t prep_msg;           /* joint-rand seed, or 0 */
  size_t prep_state;         /* out share (|| corrected joint-rand seed); private to this library */
  size_t out_share;
  size_t agg_share;
} cb200_prio3_sizes;
/* Validates cfg as above and fills *out. */
int cb200_prio3_get_sizes(const cb200_prio3_config *cfg, cb200_prio3_sizes *out);
/* PrepInit (prio3.go:245-324) of n reports under one 32-byte verify key as aggregator agg_id (0 = leader): nonces,
 * public_shares (unused without joint randomness) and input_shares (leader or helper rows by agg_id) -> prep_states
 * and prep_shares. */
int cb200_prio3_prep_init(const cb200_prio3_config *cfg, const uint8_t *verify_key, uint32_t agg_id,
                          const uint8_t *nonces, const uint8_t *public_shares, const uint8_t *input_shares,
                          uint8_t *prep_states, uint8_t *prep_shares, uint8_t *status, size_t n);
/* PrepSharesToPrep (:332-377): row i of prep_shares is the num_shares prep shares of report i, in aggregator order
 * -> prep_msgs (unused without joint randomness). */
int cb200_prio3_prep_shares_to_prep(const cb200_prio3_config *cfg, const uint8_t *prep_shares, uint8_t *prep_msgs,
                                    uint8_t *status, size_t n);
/* PrepNext (:386-403): prep_states and prep_msgs -> out_shares. */
int cb200_prio3_prep_next(const cb200_prio3_config *cfg, const uint8_t *prep_states, const uint8_t *prep_msgs,
                          uint8_t *out_shares, uint8_t *status, size_t n);
/* AggregateInit + AggregateUpdate (:408-420): agg_share = the sum mod p of the out shares of the reports whose status
 * byte is 0 (all of them when status is null).  n = 0 gives the zero agg share.  A host batch split across GPUs adds
 * the per-GPU sums on the host. */
int cb200_prio3_aggregate(const cb200_prio3_config *cfg, const uint8_t *out_shares, const uint8_t *status,
                          uint8_t *agg_share, size_t n);
/* Signer.BlindSign (pbrsa.go:350-375): blinded (n rows of kLen) -> sig = c^d' mod N under the key of metadata i.
 * status: 1 = c > N (ErrInvalidMessageLength), 2 = s^e' mod N != c (DecryptAndCheck's "rsa: internal error", also the
 * result of c = N or a wrong qinv). */
int cb200_pbrsa_blind_sign(const uint8_t *N, size_t N_len, const uint8_t *p, size_t p_len, const uint8_t *q,
                           size_t q_len, const uint8_t *qinv, size_t qinv_len, const uint8_t *blinded,
                           const uint8_t *meta, const uint64_t *meta_off, uint8_t *sig, uint8_t *status, size_t n);
/* Verifier.Verify (pbrsa.go:244-251): message i = msgs[msg_off[i] .. msg_off[i + 1]) under metadata i and sigs row i:
 * RSA-PSS-SHA-384 with a 48-byte salt over "msg" || I2OSP(len(metadata), 4) || metadata || message under (N, e').
 * status: 0 = valid, 1 = s >= N, 2 = an inconsistent EMSA-PSS encoding (both rsa.ErrVerification). */
int cb200_pbrsa_verify(const uint8_t *N, size_t N_len, const uint8_t *msgs, const uint64_t *msg_off,
                       const uint8_t *meta, const uint64_t *meta_off, const uint8_t *sigs, uint8_t *status, size_t n);

/* ---- Threshold RSA signatures (the reference's tss/rsa package, Shoup's protocol 1) ----
 * A dealer splits an RSA key into players key shares s_i, of which any threshold sign: each party computes its share
 * xi = x^(2 Delta s_i) mod N of the padded digest x (Delta = players!), and a combiner turns k >= threshold shares into
 * the standard RSA signature y with y^e = x mod N.  N (2048 to 4096 bits) and e are big-endian byte strings in host
 * memory, one key per call.  Served: 2 <= players <= 64 (the reference has no bound), u16 indices, k <= 64.  Rows are
 * kLen = ceil(bitlen(N) / 8) bytes (cb200_brsa_modulus_bytes) and on device buffers may start at any byte.  An argument
 * outside these rules or a null pointer is CB200_ERR_ARG with a message, before the device is touched. */
/* KeyShare.Sign (keyshare.go:188-256): digests (n rows of kLen, x < 2^(8 kLen), reduced mod N as Exp does) -> xi = x^E
 * mod N (n rows of kLen) for E = 2 Delta s_i (or the share's cached twoDeltaSi), a secret of at most
 * bitlen(N) - 2 + bitlen(2 Delta) bits: the constant-time exponentiation runs over that bound, in place of the
 * reference's optional blinding.  No per-op failure, so no status. */
int cb200_tssrsa_sign_share(const uint8_t *N, size_t N_len, int players, const uint8_t *E, size_t E_len,
                            const uint8_t *digests, uint8_t *xi, size_t n);
/* CombineSignShares (rsa_threshold.go:207-293) with the share parameters already checked: op i combines the k shares
 * xi[i] (k rows of kLen) of the indices idx[i] (k uint16 values in host byte order; a device idx must be 2-byte
 * aligned) for msgs row i -> sig row i.  e odd, 3 <= e < 2^32; 1 <= threshold <= players; threshold <= k <= 64.
 * status: 0, 1 = ErrInvalidCalc (an index 0, or a lambda that is not an integer), 2 = "rsa: internal error" (y^e mod N
 * != x, x taken unreduced, so x >= N always fails).  A failed op's row is all zero; the call itself returns 0. */
int cb200_tssrsa_combine(const uint8_t *N, size_t N_len, const uint8_t *e, size_t e_len, int players, int threshold,
                         int k, const uint16_t *idx, const uint8_t *xi, const uint8_t *msgs, uint8_t *sig,
                         uint8_t *status, size_t n);

/* ---- P-384 and P-521 ECDH (crypto/ecdh.P384() / P521()) ----
 * cb200_p384 / cb200_p521: the contract of cb200_p256 with 48-byte scalars and Shared outputs and 97-byte points and
 * KeyGen outputs (P-384), or 66 and 133 bytes (P-521).  A 66-byte P-521 scalar whose leading byte is above 0x01 is
 * >= n, so invalid. */
int cb200_p384(const uint8_t *scalars, const uint8_t *points, uint8_t *out, uint8_t *status, size_t n);
int cb200_p521(const uint8_t *scalars, const uint8_t *points, uint8_t *out, uint8_t *status, size_t n);

/* ---- HPKE DHKEM(P-384, HKDF-SHA384), kem_id 0x11, and DHKEM(P-521, HKDF-SHA512), kem_id 0x12 (hpke/algs.go) ----
 * The cb200_hpke_p256_* contracts, on their own entry points; the generic entry points keep treating 0x11 and 0x12 as
 * unknown.  Sizes (P-384 / P-521): seed, encapsulation seed and sk 48 / 66, pk and enc 97 / 133, ss 48 / 64.
 * keygen = DeriveKeyPair (shortkem.go:63-90): the first candidate LabeledExpand(dkp_prk, "candidate", I2OSP(ctr, 1),
 *   Nsk), with its first byte ANDed with 0xff / 0x01, that lies in [1, n - 1].  P-521's 66-byte candidate is two
 *   HKDF-Expand blocks. */
#define CB200_HPKE_P384_HKDF_SHA384 0x11
#define CB200_HPKE_P521_HKDF_SHA512 0x12
int cb200_hpke_p384_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_hpke_p384_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *seeds, uint8_t *enc, uint8_t *ss,
                           uint8_t *status, size_t n);
int cb200_hpke_p384_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, uint8_t *ss, uint8_t *status,
                           size_t n);
int cb200_hpke_p384_auth_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *skS, size_t skS_stride,
                                const uint8_t *seeds, uint8_t *enc, uint8_t *ss, uint8_t *status, size_t n);
int cb200_hpke_p384_auth_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, const uint8_t *pkS,
                                size_t pkS_stride, uint8_t *ss, uint8_t *status, size_t n);
size_t cb200_hpke_p384_public_key_size(void);             /* 97 */
size_t cb200_hpke_p384_private_key_size(void);            /* 48 */
size_t cb200_hpke_p384_ciphertext_size(void);             /* 97 */
size_t cb200_hpke_p384_shared_key_size(void);             /* 48 */
size_t cb200_hpke_p384_seed_size(void);                   /* 48 */
size_t cb200_hpke_p384_encapsulation_seed_size(void);     /* 48 */
int cb200_hpke_p521_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_hpke_p521_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *seeds, uint8_t *enc, uint8_t *ss,
                           uint8_t *status, size_t n);
int cb200_hpke_p521_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, uint8_t *ss, uint8_t *status,
                           size_t n);
int cb200_hpke_p521_auth_encaps(const uint8_t *pkR, size_t pkR_stride, const uint8_t *skS, size_t skS_stride,
                                const uint8_t *seeds, uint8_t *enc, uint8_t *ss, uint8_t *status, size_t n);
int cb200_hpke_p521_auth_decaps(const uint8_t *skR, size_t skR_stride, const uint8_t *enc, const uint8_t *pkS,
                                size_t pkS_stride, uint8_t *ss, uint8_t *status, size_t n);
size_t cb200_hpke_p521_public_key_size(void);             /* 133 */
size_t cb200_hpke_p521_private_key_size(void);            /* 66 */
size_t cb200_hpke_p521_ciphertext_size(void);             /* 133 */
size_t cb200_hpke_p521_shared_key_size(void);             /* 64 */
size_t cb200_hpke_p521_seed_size(void);                   /* 66 */
size_t cb200_hpke_p521_encapsulation_seed_size(void);     /* 66 */

/* ---- FrodoKEM-640-SHAKE (kem/frodo/frodo640shake), the only parameter set the reference has ----
 * Sizes: pk 9616, sk 19888, ct 9720, ss 16, seed 48 (s || seedSE || z), encapsulation seed 16 (mu).
 * keygen = DeriveKeyPair (frodo.go:84-135); encaps = EncapsulateDeterministically (:160-240); decaps = Decapsulate
 *   (:247-329), which never fails: a ciphertext that does not re-encrypt gives F(ct || s) (implicit rejection), and
 *   keys are not validated, as in the reference (Unpack reads any bytes).  So there is no status array.
 * Strides: 0 = one key for the whole batch.  Then A and H(pk) are computed once per call and S'A runs as one
 *   tensor-core GEMM over the batch; the bytes are the same as with the key repeated at full stride.
 * Device pointers and strides: 8-byte aligned (a contiguous batch of 9720-byte ciphertexts is not 16-byte aligned). */
int cb200_frodo640shake_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_frodo640shake_encaps(const uint8_t *pk, size_t pk_stride, const uint8_t *seeds, uint8_t *ct, uint8_t *ss,
                               size_t n);
int cb200_frodo640shake_decaps(const uint8_t *sk, size_t sk_stride, const uint8_t *ct, uint8_t *ss, size_t n);
size_t cb200_frodo640shake_public_key_size(void);
size_t cb200_frodo640shake_private_key_size(void);
size_t cb200_frodo640shake_ciphertext_size(void);
size_t cb200_frodo640shake_shared_key_size(void);
size_t cb200_frodo640shake_seed_size(void);
size_t cb200_frodo640shake_encapsulation_seed_size(void);

/* ---- ML-DSA (mode = 44, 65 or 87) and round-3 Dilithium (mode = 2, 3 or 5); sign/dilithium/gen.go:80-162 ----
 * Same contracts as the ML-DSA-65 entry points documented below, with the parameter set as first argument:
 *   ML-DSA-44 / 65 / 87 (sign/mldsa/mldsa{44,65,87}):    sk 2560 / 4032 / 4896, pk 1312 / 1952 / 2592, sig 2420 / 3309 / 4627
 *   Dilithium2 / 3 / 5  (sign/dilithium/mode{2,3,5}):     sk 2528 / 4000 / 4864, pk 1312 / 1952 / 2592, sig 2420 / 3293 / 4595
 * Round 3 (NIST = false, internal/params.go:15-17) has no context string (a non-empty one is CB200_ERR_ARG, the
 * reference's sign.ErrContextNotSupported), ignores rnd and flags, and signs the message as given. */
int cb200_mldsa_sign(int mode, const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                     const uint8_t *context, size_t ctxlen, const uint8_t *rnd, uint8_t *sig, uint8_t *status, size_t n,
                     int flags, uint64_t *attempts);
int cb200_mldsa_verify(int mode, const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                       const uint8_t *context, size_t ctxlen, const uint8_t *sig, uint8_t *ok, size_t n, int flags);
int cb200_mldsa_keygen(int mode, const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
size_t cb200_mldsa_public_key_size(int mode);
size_t cb200_mldsa_private_key_size(int mode);
size_t cb200_mldsa_signature_size(int mode);

/* ---- Ed25519 (sign/ed25519, RFC 8032 pure Ed25519) ----
 * keygen = NewKeyFromSeed (ed25519.go:206-223): seeds n x 32 -> pk n x 32, sk n x 64 (= seed || pk; may be NULL).
 * sign = Sign (ed25519.go:290-294): sk rows of 64 bytes at sk + i*sk_stride (0 = one key for the batch); A is read
 * from bytes 32..63 of the key as given, as the reference does; sig n x 64.
 * verify = Verify (ed25519.go:329-368): ok[i] = 1 iff S < L, pk decodes and encode([S]B - [k]A) == R (cofactorless).
 * Messages as in cb200_mldsa_sign (msgs back to back, n + 1 offsets, 8 bytes of read padding behind the last one).
 * The kernels read messages in aligned 8-byte words: besides the padding, a device-pointer call may read the bytes of
 * the 8-byte-aligned word that holds msgs[0] in front of it (their values are not used).
 * Device pointers: seeds, pk, sk, sig and the strides 4-byte aligned, msg_off 8-byte aligned. */
int cb200_ed25519_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_ed25519_sign(const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *sig,
                       size_t n);
int cb200_ed25519_verify(const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                         const uint8_t *sig, uint8_t *ok, size_t n);
size_t cb200_ed25519_public_key_size(void);  /* 32 */
size_t cb200_ed25519_private_key_size(void); /* 64 */
size_t cb200_ed25519_signature_size(void);   /* 64 */
size_t cb200_ed25519_seed_size(void);        /* 32 */

/* ---- Ed25519-Dilithium2 (sign/eddilithium2): pk = Dilithium2 pk (1312) || Ed25519 pk (32) = 1344, sk = Dilithium2
 * packed sk (2528) || Ed25519 seed (32) = 2560, sig = Dilithium2 sig (2420) || Ed25519 sig (64) = 2484, seed 32.
 * keygen = NewKeyFromSeed (eddilithium.go:59-78, SHAKE256(seed) -> Dilithium2 seed || Ed25519 seed); sign = SignTo
 * (:82-93; the Ed25519 public key is re-derived from the seed, as PrivateKey.Unpack does); verify = Verify (:96-115,
 * both halves).  status (optional): 1 = Dilithium2's 576-attempt cap (CB200_ERR_SIGN_ATTEMPTS for host pointers).
 * No context string (sign.ErrContextNotSupported).  Device pointers: seeds, pk, sk, their strides and msg_off 16-byte
 * aligned; sig 4-byte aligned (its Ed25519 half starts at byte 2420). */
int cb200_eddilithium2_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_eddilithium2_sign(const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *sig,
                            uint8_t *status, size_t n);
int cb200_eddilithium2_verify(const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                              const uint8_t *sig, uint8_t *ok, size_t n);
size_t cb200_eddilithium2_public_key_size(void);  /* 1344 */
size_t cb200_eddilithium2_private_key_size(void); /* 2560 */
size_t cb200_eddilithium2_signature_size(void);   /* 2484 */
size_t cb200_eddilithium2_seed_size(void);        /* 32 */

/* ---- Ed448 (sign/ed448, RFC 8032 pure Ed448) ----
 * keygen = NewKeyFromSeed (ed448.go:191-205): seeds n x 57 -> pk n x 57, sk n x 114 (= seed || pk; may be NULL).
 * sign = Sign (ed448.go:207-271): sk rows of 114 bytes at sk + i*sk_stride (0 = one key for the batch); A is read from
 * bytes 57..113 of the key as given, as the reference does; sig n x 114.
 * verify = Verify (ed448.go:294-339): ok[i] = 1 iff S < l with byte 113 = 0, pk decodes and encode(Q) == R for the
 * reference's Q = [S]G - [4 ((k / 4) mod l)]A, which drops the 4-torsion component of A.
 * context: one host string of ctxlen bytes for the whole batch (may be NULL when ctxlen = 0).  ctxlen > 255: sign
 * returns CB200_ERR_ARG (the reference panics), verify sets every ok[i] = 0 and returns 0 (the reference returns false).
 * Messages as in cb200_ed25519_sign, with the same read rule around msgs[0] and behind the last message.
 * Device pointers: msg_off 8-byte aligned; seeds, keys and signatures may start at any byte. */
int cb200_ed448_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_ed448_sign(const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                     const uint8_t *context, size_t ctxlen, uint8_t *sig, size_t n);
int cb200_ed448_verify(const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                       const uint8_t *context, size_t ctxlen, const uint8_t *sig, uint8_t *ok, size_t n);
size_t cb200_ed448_public_key_size(void);  /* 57 */
size_t cb200_ed448_private_key_size(void); /* 114 */
size_t cb200_ed448_signature_size(void);   /* 114 */
size_t cb200_ed448_seed_size(void);        /* 57 */

/* ---- Ed448-Dilithium3 (sign/eddilithium3): pk = Dilithium3 pk (1952) || Ed448 pk (57) = 2009, sk = Dilithium3
 * packed sk (4000) || Ed448 seed (57) = 4057, sig = Dilithium3 sig (3293) || Ed448 sig (114) = 3407, seed 57.
 * keygen = NewKeyFromSeed (eddilithium.go:59-78, SHAKE256(seed) -> Dilithium3 seed (32) || Ed448 seed (57)); sign =
 * SignTo (:82-93; Ed448 with an empty context, its public key re-derived from the seed as PrivateKey.Unpack does);
 * verify = Verify (:96-110, both halves).  status (optional): 1 = Dilithium3's 576-attempt cap (CB200_ERR_SIGN_ATTEMPTS
 * for host pointers).  No context string (sign.ErrContextNotSupported).  Device pointers: msg_off 16-byte aligned
 * (the Dilithium3 flows read it); seeds, keys, signatures and strides may be at any byte, since every row size is odd
 * and the Dilithium3 halves are staged through aligned scratch. */
int cb200_eddilithium3_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
int cb200_eddilithium3_sign(const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off, uint8_t *sig,
                            uint8_t *status, size_t n);
int cb200_eddilithium3_verify(const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                              const uint8_t *sig, uint8_t *ok, size_t n);
size_t cb200_eddilithium3_public_key_size(void);  /* 2009 */
size_t cb200_eddilithium3_private_key_size(void); /* 4057 */
size_t cb200_eddilithium3_signature_size(void);   /* 3407 */
size_t cb200_eddilithium3_seed_size(void);        /* 57 */

/* ---- ML-DSA-65 ---- */
/* sign.Scheme.Sign / SignTo    sign/mldsa/mldsa65/dilithium.go:282-303,56-84  ->
 * internal.SignTo (ML-DSA.Sign_internal)  sign/mldsa/mldsa65/internal/dilithium.go:340-470,
 * including (*PrivateKey).Unpack (:142-163): A = ExpandA(rho), NTT(s1), NTT(s2), NTT(t0) are rebuilt on
 * the device (once if sk_stride = 0, else per operation).
 * sk: packed private key(s), 4032 bytes; op i uses sk + i*sk_stride (0 = one key for all).
 * msgs: all messages back to back; message i = msgs[msg_off[i] .. msg_off[i+1]) (n+1 offsets).
 * context/ctxlen: the FIPS 204 context string, shared by the batch (ctxlen <= 255; host pointer).
 * rnd: n x 32 bytes of signing randomness, or NULL for deterministic signing (rnd = 0^32).
 * sig: n x 3309 bytes.  status (optional): n bytes, 1 = the 576-attempt cap was hit (the reference
 * panics there); attempts (optional, host pointer): total rejection-loop iterations of the batch.
 * flags: CB200_SIGN_INTERNAL = ML-DSA.Sign_internal on the message as given (no 0x00||len||ctx framing,
 * the ACVP interface, sign/mldsa/mldsa65/dilithium.go:87-98). */
int cb200_mldsa65_sign(const uint8_t *sk, size_t sk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                       const uint8_t *context, size_t ctxlen, const uint8_t *rnd, uint8_t *sig, uint8_t *status,
                       size_t n, int flags, uint64_t *attempts);
/* sign.Scheme.Verify       sign/mldsa/mldsa65/dilithium.go:305-330,115-138 -> internal.Verify internal/dilithium.go:273-332,
 * including (*PublicKey).Unpack (:113-126): A = ExpandA(rho), tr = H(pk) rebuilt on the device.
 * pk: packed public key(s), 1952 bytes, op i uses pk + i*pk_stride (0 = shared); sig: n x 3309 bytes;
 * ok: n bytes, 1 = valid.  A signature of the wrong length is the caller's (shim's) `false`. */
int cb200_mldsa65_verify(const uint8_t *pk, size_t pk_stride, const uint8_t *msgs, const uint64_t *msg_off,
                         const uint8_t *context, size_t ctxlen, const uint8_t *sig, uint8_t *ok, size_t n, int flags);
/* sign.Scheme.DeriveKey    sign/mldsa/mldsa65/dilithium.go:266-276 -> internal.NewKeyFromSeed internal/dilithium.go:181-241.
 * seeds: n x 32; pk: n x 1952; sk: n x 4032 (packed, = MarshalBinary). */
int cb200_mldsa65_keygen(const uint8_t *seeds, uint8_t *pk, uint8_t *sk, size_t n);
size_t cb200_mldsa65_public_key_size(void);
size_t cb200_mldsa65_signature_size(void);
size_t cb200_mldsa65_private_key_size(void);

#ifdef __cplusplus
}
#endif
#endif
