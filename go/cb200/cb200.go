//go:build cuda && cgo

// Package cb200 is the cgo binding of libcirclb200.so (include/circl_b200.h):
// the cb200 batch engine for CIRCL's module-lattice hot path.
//
// NOTE: this file is delivered as source.  The build image has no Go toolchain
// (`go version` fails), so it is reviewed, not compiled, here; every executable
// test and timing drives the same C ABI from Python/C (see INTEGRATION.md).
package cb200

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../circl_b200 -lcirclb200 -Wl,-rpath,${SRCDIR}/../../circl_b200
#include <stdlib.h>
#include "circl_b200.h"
*/
import "C"

import (
	"errors"
	"runtime"
	"sync"
	"unsafe"
)

// Errors mirror the negative codes of the C ABI.
var (
	ErrNotInit = errors.New("cb200: not initialised / no CUDA device")
	ErrPubKey  = errors.New("cb200: encapsulation key is not canonical") // mapped to kem.ErrPubKey by callers
	ErrPrivKey = errors.New("cb200: H(ek) stored in the decapsulation key does not match") // kem.ErrPrivKey
)

var initOnce sync.Once
var initErr error

// Init drives every visible GPU from this process (cb200_init_devices(0)): host-slice batches are cut into one
// contiguous index range per GPU inside the library and the results land in the caller's slices in index order, so a
// kem.Scheme / sign.Scheme caller never sees devices.  Safe to call many times and from any goroutine.
func Init() error { return InitDevices(0) }

// InitDevices restricts the library to GPUs 0..ndev-1 (ndev <= 0: all).
func InitDevices(ndev int) error {
	initOnce.Do(func() {
		initErr = call(func() C.int { return C.cb200_init_devices(C.int(ndev)) })
	})
	return initErr
}

// ActiveDevices reports how many GPUs the library drives (0 before Init).
func ActiveDevices() int { return int(C.cb200_active_devices()) }

// call runs one C entry point and turns its return code into an error.  cb200_last_error() is per OS thread and a
// goroutine may migrate between two cgo calls, so the call and the error fetch are pinned to one thread.
func call(f func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return lastErr(f())
}

// lastErr must run on the OS thread that made the failing call (see call).
func lastErr(rc C.int) error {
	switch rc {
	case 0:
		return nil
	case C.CB200_ERR_PUBKEY:
		return ErrPubKey
	case C.CB200_ERR_PRIVKEY:
		return ErrPrivKey
	case C.CB200_ERR_NOT_INIT:
		return ErrNotInit
	case C.CB200_ERR_ARG:
		// programmer error: the reference panics on wrong lengths (kem/mlkem/mlkem768/kyber.go:110-121)
		panic(C.GoString(C.cb200_last_error()))
	}
	return errors.New(C.GoString(C.cb200_last_error()))
}

// KyberNTT runs (*Poly).NTT (inverse=false) or InvNTT on every polynomial, in place.
// Replaces nttAVX2 / invNttAVX2 (pke/kyber/internal/common/stubs_amd64.go:8-14) for batches.
// The slice is caller-owned; the library does not retain the pointer past the call (cgo rule).
func KyberNTT(polys [][256]int16, inverse bool) error {
	if len(polys) == 0 {
		return nil
	}
	inv := C.int(0)
	if inverse {
		inv = 1
	}
	return call(func() C.int {
		return C.cb200_kyber_ntt((*C.int16_t)(unsafe.Pointer(&polys[0])), C.size_t(len(polys)), inv)
	})
}

// KyberMulHat: p[i] = a[i] (*) b[i]  (mulHatAVX2, stubs_amd64.go:17).
func KyberMulHat(p, a, b [][256]int16) error {
	if len(p) != len(a) || len(p) != len(b) {
		panic("cb200: length mismatch")
	}
	if len(p) == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_kyber_mulhat((*C.int16_t)(unsafe.Pointer(&p[0])), (*C.int16_t)(unsafe.Pointer(&a[0])),
		(*C.int16_t)(unsafe.Pointer(&b[0])), C.size_t(len(p)))
	})
}

// DilithiumNTT: (*Poly).NTT / InvNTT of sign/internal/dilithium over a batch, in place.
func DilithiumNTT(polys [][256]uint32, inverse bool) error {
	if len(polys) == 0 {
		return nil
	}
	inv := C.int(0)
	if inverse {
		inv = 1
	}
	return call(func() C.int {
		return C.cb200_dil_ntt((*C.uint32_t)(unsafe.Pointer(&polys[0])), C.size_t(len(polys)), inv)
	})
}

// MLKEMEncaps: batched UnmarshalBinaryPublicKey + EncapsulateDeterministically.
// k = 3 (ML-KEM-768) or 4 (ML-KEM-1024).  ek holds either one packed key (shared) or
// n keys back to back; seeds is n*32 bytes.  ct and ss are written in place.
func MLKEMEncaps(k int, ek []byte, shared bool, seeds, ct, ss []byte) error {
	n := len(seeds) / 32
	ekSize := int(C.cb200_mlkem_public_key_size(C.int(k)))
	ctSize := int(C.cb200_mlkem_ciphertext_size(C.int(k)))
	stride := C.size_t(ekSize)
	if shared {
		stride = 0
		if len(ek) != ekSize {
			panic("cb200: ek must be one packed key")
		}
	} else if len(ek) != n*ekSize {
		panic("cb200: ek must hold n packed keys")
	}
	if len(ct) != n*ctSize || len(ss) != n*32 {
		panic("cb200: ct/ss have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_mlkem_encaps(C.int(k), (*C.uint8_t)(unsafe.Pointer(&ek[0])), stride,
		(*C.uint8_t)(unsafe.Pointer(&seeds[0])), (*C.uint8_t)(unsafe.Pointer(&ct[0])),
		(*C.uint8_t)(unsafe.Pointer(&ss[0])), nil, C.size_t(n))
	})
}

// MLKEMDecaps: batched UnmarshalBinaryPrivateKey + Decapsulate (implicit rejection included).
func MLKEMDecaps(k int, dk []byte, shared bool, ct, ss []byte) error {
	dkSize := int(C.cb200_mlkem_private_key_size(C.int(k)))
	ctSize := int(C.cb200_mlkem_ciphertext_size(C.int(k)))
	n := len(ct) / ctSize
	stride := C.size_t(dkSize)
	if shared {
		stride = 0
	}
	if len(ct) != n*ctSize || len(ss) != n*32 || (shared && len(dk) != dkSize) || (!shared && len(dk) != n*dkSize) {
		panic("cb200: dk/ct/ss have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_mlkem_decaps(C.int(k), (*C.uint8_t)(unsafe.Pointer(&dk[0])), stride,
		(*C.uint8_t)(unsafe.Pointer(&ct[0])), (*C.uint8_t)(unsafe.Pointer(&ss[0])), nil, C.size_t(n))
	})
}

// MLDSA65Sign signs len(msgs) messages.  sk holds one packed 4032-byte key (shared) or one per message.
// rnd == nil selects deterministic signing (sign/mldsa/mldsa65/dilithium.go:57-63).  ctx must be <= 255 bytes
// (the caller returns sign.ErrContextTooLong otherwise).  sig receives len(msgs)*3309 bytes.
func MLDSA65Sign(sk []byte, shared bool, msgs [][]byte, ctx, rnd, sig []byte) error {
	n := len(msgs)
	if n == 0 {
		return nil
	}
	off := make([]uint64, n+1)
	total := 0
	for i, m := range msgs {
		off[i] = uint64(total)
		total += len(m)
	}
	off[n] = uint64(total)
	blob := make([]byte, total+8)
	for i, m := range msgs {
		copy(blob[off[i]:], m)
	}
	stride := C.size_t(4032)
	if shared {
		stride = 0
	}
	var pctx, prnd *C.uint8_t
	if len(ctx) > 0 {
		pctx = (*C.uint8_t)(unsafe.Pointer(&ctx[0]))
	}
	if rnd != nil {
		prnd = (*C.uint8_t)(unsafe.Pointer(&rnd[0]))
	}
	return call(func() C.int {
		return C.cb200_mldsa65_sign((*C.uint8_t)(unsafe.Pointer(&sk[0])), stride,
		(*C.uint8_t)(unsafe.Pointer(&blob[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])), pctx, C.size_t(len(ctx)),
		prnd, (*C.uint8_t)(unsafe.Pointer(&sig[0])), nil, C.size_t(n), 0, nil)
	})
}

// packMsgs lays messages back to back with n+1 offsets and the 8 bytes of read padding the sign entry points need.
func packMsgs(msgs [][]byte) ([]byte, []uint64) {
	n := len(msgs)
	off := make([]uint64, n+1)
	total := 0
	for i, m := range msgs {
		off[i] = uint64(total)
		total += len(m)
	}
	off[n] = uint64(total)
	blob := make([]byte, total+8)
	for i, m := range msgs {
		copy(blob[off[i]:], m)
	}
	return blob, off
}

func u8(b []byte) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(&b[0])) }

// Ed25519KeyGen: ed25519.NewKeyFromSeed (sign/ed25519/ed25519.go:206-223) on n 32-byte seeds; pk receives n*32
// bytes, sk n*64 (seed || public key).
func Ed25519KeyGen(seeds, pk, sk []byte) error {
	n := len(seeds) / 32
	if len(seeds) != n*32 || len(pk) != n*32 || len(sk) != n*64 {
		panic("cb200: seeds/pk/sk have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_ed25519_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// Ed25519SignBatch: ed25519.Sign (ed25519.go:290-294) on len(msgs) messages.  sk holds one 64-byte private key
// (shared) or one per message; its public half is used as given.  sig receives len(msgs)*64 bytes.
func Ed25519SignBatch(sk []byte, shared bool, msgs [][]byte, sig []byte) error {
	n := len(msgs)
	if (shared && len(sk) != 64) || (!shared && len(sk) != n*64) || len(sig) != n*64 {
		panic("cb200: sk/sig have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	stride := C.size_t(64)
	if shared {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_ed25519_sign(u8(sk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig), C.size_t(n))
	})
}

// Ed25519VerifyBatch: ed25519.Verify (ed25519.go:329-368) on len(msgs) 64-byte signatures; pk holds one 32-byte public
// key (shared) or one per message.  ok[i] is the reference's result.
func Ed25519VerifyBatch(pk []byte, shared bool, msgs [][]byte, sig []byte, ok []bool) error {
	n := len(msgs)
	if (shared && len(pk) != 32) || (!shared && len(pk) != n*32) || len(sig) != n*64 || len(ok) != n {
		panic("cb200: pk/sig/ok have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return verifyBatch(n, msgs, ok, func(blob []byte, off []uint64, res []byte) C.int {
		stride := C.size_t(32)
		if shared {
			stride = 0
		}
		return C.cb200_ed25519_verify(u8(pk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig), u8(res),
			C.size_t(n))
	})
}

func verifyBatch(n int, msgs [][]byte, ok []bool, f func(blob []byte, off []uint64, res []byte) C.int) error {
	blob, off := packMsgs(msgs)
	res := make([]byte, n)
	if err := call(func() C.int { return f(blob, off, res) }); err != nil {
		return err
	}
	for i := range ok {
		ok[i] = res[i] != 0
	}
	return nil
}

// Sizes of Ed25519-Dilithium2 (sign/eddilithium2/eddilithium.go:16-28).
const (
	EdDilithium2PublicKeySize  = 1344
	EdDilithium2PrivateKeySize = 2560
	EdDilithium2SignatureSize  = 2484
)

// EdDilithium2KeyGen: eddilithium2.NewKeyFromSeed (eddilithium.go:59-78) on n 32-byte seeds; pk and sk receive the
// packed keys (n*1344 and n*2560 bytes).
func EdDilithium2KeyGen(seeds, pk, sk []byte) error {
	n := len(seeds) / 32
	if len(seeds) != n*32 || len(pk) != n*EdDilithium2PublicKeySize || len(sk) != n*EdDilithium2PrivateKeySize {
		panic("cb200: seeds/pk/sk have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_eddilithium2_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// EdDilithium2SignBatch: eddilithium2.SignTo (eddilithium.go:82-93) on len(msgs) messages with one packed key
// (shared) or one per message; sig receives len(msgs)*2484 bytes.  An error is returned if a Dilithium2 half
// exhausted its 576 attempts (the reference panics there).
func EdDilithium2SignBatch(sk []byte, shared bool, msgs [][]byte, sig []byte) error {
	n := len(msgs)
	if (shared && len(sk) != EdDilithium2PrivateKeySize) || (!shared && len(sk) != n*EdDilithium2PrivateKeySize) ||
		len(sig) != n*EdDilithium2SignatureSize {
		panic("cb200: sk/sig have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	stride := C.size_t(EdDilithium2PrivateKeySize)
	if shared {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_eddilithium2_sign(u8(sk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig), nil,
			C.size_t(n))
	})
}

// EdDilithium2VerifyBatch: eddilithium2.Verify (eddilithium.go:96-115): both halves must verify.
func EdDilithium2VerifyBatch(pk []byte, shared bool, msgs [][]byte, sig []byte, ok []bool) error {
	n := len(msgs)
	if (shared && len(pk) != EdDilithium2PublicKeySize) || (!shared && len(pk) != n*EdDilithium2PublicKeySize) ||
		len(sig) != n*EdDilithium2SignatureSize || len(ok) != n {
		panic("cb200: pk/sig/ok have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return verifyBatch(n, msgs, ok, func(blob []byte, off []uint64, res []byte) C.int {
		stride := C.size_t(EdDilithium2PublicKeySize)
		if shared {
			stride = 0
		}
		return C.cb200_eddilithium2_verify(u8(pk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig),
			u8(res), C.size_t(n))
	})
}

// ctxPtr returns a pointer to the context bytes (nil for an empty context).
func ctxPtr(ctx []byte) *C.uint8_t {
	if len(ctx) == 0 {
		return nil
	}
	return u8(ctx)
}

// Ed448KeyGen: ed448.NewKeyFromSeed (sign/ed448/ed448.go:191-205) on n 57-byte seeds; pk receives n*57 bytes, sk
// n*114 (seed || public key).
func Ed448KeyGen(seeds, pk, sk []byte) error {
	n := len(seeds) / 57
	if len(seeds) != n*57 || len(pk) != n*57 || len(sk) != n*114 {
		panic("cb200: seeds/pk/sk have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_ed448_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// Ed448SignBatch: ed448.Sign (ed448.go:207-271) on len(msgs) messages with the context ctx (at most 255 bytes; longer
// returns an error where the reference panics).  sk holds one 114-byte private key (shared) or one per message; its
// public half is used as given.  sig receives len(msgs)*114 bytes.
func Ed448SignBatch(sk []byte, shared bool, msgs [][]byte, ctx []byte, sig []byte) error {
	n := len(msgs)
	if (shared && len(sk) != 114) || (!shared && len(sk) != n*114) || len(sig) != n*114 {
		panic("cb200: sk/sig have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	stride := C.size_t(114)
	if shared {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_ed448_sign(u8(sk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), ctxPtr(ctx),
			C.size_t(len(ctx)), u8(sig), C.size_t(n))
	})
}

// Ed448VerifyBatch: ed448.Verify (ed448.go:294-339) on len(msgs) 114-byte signatures with the context ctx; pk holds
// one 57-byte public key (shared) or one per message.  ok[i] is the reference's result (all false for a context over
// 255 bytes).
func Ed448VerifyBatch(pk []byte, shared bool, msgs [][]byte, ctx []byte, sig []byte, ok []bool) error {
	n := len(msgs)
	if (shared && len(pk) != 57) || (!shared && len(pk) != n*57) || len(sig) != n*114 || len(ok) != n {
		panic("cb200: pk/sig/ok have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return verifyBatch(n, msgs, ok, func(blob []byte, off []uint64, res []byte) C.int {
		stride := C.size_t(57)
		if shared {
			stride = 0
		}
		return C.cb200_ed448_verify(u8(pk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), ctxPtr(ctx),
			C.size_t(len(ctx)), u8(sig), u8(res), C.size_t(n))
	})
}

// Sizes of Ed448-Dilithium3 (sign/eddilithium3/eddilithium.go:16-28).
const (
	EdDilithium3PublicKeySize  = 2009
	EdDilithium3PrivateKeySize = 4057
	EdDilithium3SignatureSize  = 3407
)

// EdDilithium3KeyGen: eddilithium3.NewKeyFromSeed (eddilithium.go:59-78) on n 57-byte seeds; pk and sk receive the
// packed keys (n*2009 and n*4057 bytes).
func EdDilithium3KeyGen(seeds, pk, sk []byte) error {
	n := len(seeds) / 57
	if len(seeds) != n*57 || len(pk) != n*EdDilithium3PublicKeySize || len(sk) != n*EdDilithium3PrivateKeySize {
		panic("cb200: seeds/pk/sk have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_eddilithium3_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// EdDilithium3SignBatch: eddilithium3.SignTo (eddilithium.go:82-93) on len(msgs) messages with one packed key
// (shared) or one per message; sig receives len(msgs)*3407 bytes.  An error is returned if a Dilithium3 half
// exhausted its 576 attempts (the reference panics there).
func EdDilithium3SignBatch(sk []byte, shared bool, msgs [][]byte, sig []byte) error {
	n := len(msgs)
	if (shared && len(sk) != EdDilithium3PrivateKeySize) || (!shared && len(sk) != n*EdDilithium3PrivateKeySize) ||
		len(sig) != n*EdDilithium3SignatureSize {
		panic("cb200: sk/sig have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	stride := C.size_t(EdDilithium3PrivateKeySize)
	if shared {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_eddilithium3_sign(u8(sk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig), nil,
			C.size_t(n))
	})
}

// EdDilithium3VerifyBatch: eddilithium3.Verify (eddilithium.go:96-110): both halves must verify.
func EdDilithium3VerifyBatch(pk []byte, shared bool, msgs [][]byte, sig []byte, ok []bool) error {
	n := len(msgs)
	if (shared && len(pk) != EdDilithium3PublicKeySize) || (!shared && len(pk) != n*EdDilithium3PublicKeySize) ||
		len(sig) != n*EdDilithium3SignatureSize || len(ok) != n {
		panic("cb200: pk/sig/ok have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return verifyBatch(n, msgs, ok, func(blob []byte, off []uint64, res []byte) C.int {
		stride := C.size_t(EdDilithium3PublicKeySize)
		if shared {
			stride = 0
		}
		return C.cb200_eddilithium3_verify(u8(pk), stride, u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig),
			u8(res), C.size_t(n))
	})
}

// Hybrid scheme identifiers of include/circl_b200.h (kem/hybrid/hybrid.go:34-93).
const (
	HybridX25519MLKEM768 = 0
	HybridKyber768X25519 = 1
	HybridKyber512X25519 = 2
	HybridKyber768X448   = 3
	HybridKyber1024X448  = 4
)

// X25519Batch: x25519.KeyGen (points == nil) or x25519.Shared (dh/x25519/key.go:44-56) on n 32-byte keys.
// ok[i] is false where Shared would have returned false (point of small order); out[i] is then all zero.
func X25519Batch(scalars, points, out []byte, ok []bool) error {
	n := len(scalars) / 32
	if len(out) != n*32 || (points != nil && len(points) != n*32) || (ok != nil && len(ok) != n) {
		panic("cb200: X25519Batch buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	status := make([]byte, n)
	var pp *C.uint8_t
	if points != nil {
		pp = (*C.uint8_t)(unsafe.Pointer(&points[0]))
	}
	var rc C.int
	err := call(func() C.int {
		rc = C.cb200_x25519((*C.uint8_t)(unsafe.Pointer(&scalars[0])), pp, (*C.uint8_t)(unsafe.Pointer(&out[0])),
			(*C.uint8_t)(unsafe.Pointer(&status[0])), C.size_t(n))
		if rc == C.CB200_ERR_PUBKEY { // reported per operation through ok, like the bool of x25519.Shared
			return 0
		}
		return rc
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

// X448Batch: x448.KeyGen (points == nil) or x448.Shared (dh/x448/key.go:33-46) on n 56-byte keys.
// ok[i] is false where Shared would have returned false (low-order point); out[i] is then all zero.
func X448Batch(scalars, points, out []byte, ok []bool) error {
	n := len(scalars) / 56
	if len(out) != n*56 || (points != nil && len(points) != n*56) || (ok != nil && len(ok) != n) {
		panic("cb200: X448Batch buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	status := make([]byte, n)
	var pp *C.uint8_t
	if points != nil {
		pp = (*C.uint8_t)(unsafe.Pointer(&points[0]))
	}
	var rc C.int
	err := call(func() C.int {
		rc = C.cb200_x448((*C.uint8_t)(unsafe.Pointer(&scalars[0])), pp, (*C.uint8_t)(unsafe.Pointer(&out[0])),
			(*C.uint8_t)(unsafe.Pointer(&status[0])), C.size_t(n))
		if rc == C.CB200_ERR_PUBKEY { // reported per operation through ok, like the bool of x448.Shared
			return 0
		}
		return rc
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

// XWingEncaps: batched xwing.Encapsulate (kem/xwing/xwing.go:173-182).  pk: one packed 1216-byte key (shared) or n keys;
// seeds: n*64 bytes; ct: n*1120; ss: n*32.  kem.ErrPubKey is returned if any ML-KEM half is not canonical.
func XWingEncaps(pk []byte, shared bool, seeds, ct, ss []byte) error {
	n := len(seeds) / 64
	stride := C.size_t(1216)
	if shared {
		stride = 0
	}
	if len(ct) != n*1120 || len(ss) != n*32 || (shared && len(pk) != 1216) || (!shared && len(pk) != n*1216) {
		panic("cb200: XWingEncaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_xwing_encaps((*C.uint8_t)(unsafe.Pointer(&pk[0])), stride, (*C.uint8_t)(unsafe.Pointer(&seeds[0])),
		(*C.uint8_t)(unsafe.Pointer(&ct[0])), (*C.uint8_t)(unsafe.Pointer(&ss[0])), nil, C.size_t(n))
	})
}

// HybridEncaps: batched hybrid.scheme.EncapsulateDeterministically (kem/hybrid/hybrid.go:233-261); id is one of the
// Hybrid* constants; seeds: n*EncapsulationSeedSize bytes (32, or 56 for the X448 hybrids); ss: n*SharedKeySize
// bytes (64, or 88 for the X448 hybrids: the two shared secrets side by side, hybrid.go:260).
func HybridEncaps(id int, pk []byte, shared bool, seeds, ct, ss []byte) error {
	seedSize := int(C.cb200_hybrid_encapsulation_seed_size(C.int(id)))
	ssSize := int(C.cb200_hybrid_shared_key_size(C.int(id)))
	if seedSize == 0 {
		panic("cb200: HybridEncaps: unknown scheme id")
	}
	n := len(seeds) / seedSize
	pkSize := int(C.cb200_hybrid_public_key_size(C.int(id)))
	ctSize := int(C.cb200_hybrid_ciphertext_size(C.int(id)))
	stride := C.size_t(pkSize)
	if shared {
		stride = 0
	}
	if len(ct) != n*ctSize || len(ss) != n*ssSize || (shared && len(pk) != pkSize) || (!shared && len(pk) != n*pkSize) {
		panic("cb200: HybridEncaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_hybrid_encaps(C.int(id), (*C.uint8_t)(unsafe.Pointer(&pk[0])), stride,
		(*C.uint8_t)(unsafe.Pointer(&seeds[0])), (*C.uint8_t)(unsafe.Pointer(&ct[0])), (*C.uint8_t)(unsafe.Pointer(&ss[0])),
		nil, C.size_t(n))
	})
}

// HPKE DHKEM identifiers of include/circl_b200.h: the HPKE KEM ids themselves (hpke/algs.go:248-277).
const (
	HPKEX25519HKDFSHA256 = 0x20
	HPKEX448HKDFSHA512   = 0x21
)

// hpkeSizes returns (N, ss) of a DHKEM id: N = key, enc and seed bytes (32 or 56), ss = shared secret bytes (32 or 64).
func hpkeSizes(id int, fn string) (int, int) {
	n := int(C.cb200_hpke_public_key_size(C.int(id)))
	if n == 0 {
		panic("cb200: " + fn + ": unknown HPKE KEM id")
	}
	return n, int(C.cb200_hpke_shared_key_size(C.int(id)))
}

// hpkeKey checks one key argument: a single key (shared by the batch, stride 0) or n keys back to back.  The
// FrodoKEM calls use it too.
func hpkeKey(k []byte, n, size int, fn string) (*C.uint8_t, C.size_t) {
	switch len(k) {
	case size:
		return u8(k), 0
	case n * size:
		return u8(k), C.size_t(size)
	}
	panic("cb200: " + fn + ": key buffer has the wrong length")
}

// HPKEKeygen: batched DeriveKeyPair (hpke/xkem.go:55-71) on n seeds of N bytes; pk and sk: n*N bytes (sk unclamped).
func HPKEKeygen(id int, seeds, pk, sk []byte) error {
	N, _ := hpkeSizes(id, "HPKEKeygen")
	n := len(seeds) / N
	if len(seeds) != n*N || len(pk) != n*N || len(sk) != n*N {
		panic("cb200: HPKEKeygen buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_hpke_keygen(C.int(id), u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// HPKEEncaps: batched Encap, or AuthEncap when skS is not nil (hpke/kembase.go:120-183).  pkR and skS: one key or
// n keys each; seeds and enc: n*N bytes; ss: n*SharedKeySize.  ErrPubKey (hpke.ErrInvalidKEMSharedSecret for the
// caller) is returned after the whole batch ran if any operation met a low-order point; ok[i] (may be nil) tells which.
func HPKEEncaps(id int, pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	N, S := hpkeSizes(id, "HPKEEncaps")
	n := len(seeds) / N
	if len(seeds) != n*N || len(enc) != n*N || len(ss) != n*S || (ok != nil && len(ok) != n) {
		panic("cb200: HPKEEncaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	pr, prs := hpkeKey(pkR, n, N, "HPKEEncaps")
	status := make([]byte, n)
	err := call(func() C.int {
		if skS == nil {
			return C.cb200_hpke_encaps(C.int(id), pr, prs, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
		}
		sp, sps := hpkeKey(skS, n, N, "HPKEEncaps")
		return C.cb200_hpke_auth_encaps(C.int(id), pr, prs, sp, sps, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

// HPKEDecaps: batched Decap, or AuthDecap when pkS is not nil (hpke/kembase.go:185-241).  skR and pkS: one key or n
// keys each (a single skR has its public key computed once); enc: n*N bytes; ss: n*SharedKeySize.  Errors as HPKEEncaps.
func HPKEDecaps(id int, skR, enc, pkS, ss []byte, ok []bool) error {
	N, S := hpkeSizes(id, "HPKEDecaps")
	n := len(enc) / N
	if len(enc) != n*N || len(ss) != n*S || (ok != nil && len(ok) != n) {
		panic("cb200: HPKEDecaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	sr, srs := hpkeKey(skR, n, N, "HPKEDecaps")
	status := make([]byte, n)
	err := call(func() C.int {
		if pkS == nil {
			return C.cb200_hpke_decaps(C.int(id), sr, srs, u8(enc), u8(ss), u8(status), C.size_t(n))
		}
		pp, pps := hpkeKey(pkS, n, N, "HPKEDecaps")
		return C.cb200_hpke_auth_decaps(C.int(id), sr, srs, u8(enc), pp, pps, u8(ss), u8(status), C.size_t(n))
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

// The NIST DHKEMs (hpke/shortkem.go; include/circl_b200.h cb200_hpke_p256_* / p384_* / p521_*), each on entry points
// of its own; the generic HPKE* functions above do not take these ids.
//   DHKEM(P-256, HKDF-SHA256), kem_id 0x10: sk and seeds 32 bytes, pk and enc 65 (0x04 || X || Y), ss 32
//   DHKEM(P-384, HKDF-SHA384), kem_id 0x11: sk and seeds 48 bytes, pk and enc 97, ss 48
//   DHKEM(P-521, HKDF-SHA512), kem_id 0x12: sk and seeds 66 bytes, pk and enc 133, ss 64
const (
	HPKEP256HKDFSHA256     = 0x10
	HPKEP256PrivateKeySize = 32
	HPKEP256PublicKeySize  = 65
	HPKEP256SharedKeySize  = 32

	HPKEP384HKDFSHA384     = 0x11
	HPKEP384PrivateKeySize = 48
	HPKEP384PublicKeySize  = 97
	HPKEP384SharedKeySize  = 48

	HPKEP521HKDFSHA512     = 0x12
	HPKEP521PrivateKeySize = 66
	HPKEP521PublicKeySize  = 133
	HPKEP521SharedKeySize  = 64
)

// nist: one NIST DHKEM's id, sizes and the prefix of its Go names (for panics)
type nist struct {
	id, sk, pk, ss int
	name           string
}

var (
	nistP256 = nist{HPKEP256HKDFSHA256, HPKEP256PrivateKeySize, HPKEP256PublicKeySize, HPKEP256SharedKeySize, "HPKEP256"}
	nistP384 = nist{HPKEP384HKDFSHA384, HPKEP384PrivateKeySize, HPKEP384PublicKeySize, HPKEP384SharedKeySize, "HPKEP384"}
	nistP521 = nist{HPKEP521HKDFSHA512, HPKEP521PrivateKeySize, HPKEP521PublicKeySize, HPKEP521SharedKeySize, "HPKEP521"}
)

func (c nist) keygen(seeds, pk, sk []byte) error {
	n := len(seeds) / c.sk
	if len(seeds) != n*c.sk || len(pk) != n*c.pk || len(sk) != n*c.sk {
		panic("cb200: " + c.name + "Keygen buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		switch c.id {
		case HPKEP384HKDFSHA384:
			return C.cb200_hpke_p384_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n))
		case HPKEP521HKDFSHA512:
			return C.cb200_hpke_p521_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n))
		}
		return C.cb200_hpke_p256_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n))
	})
}

func (c nist) encaps(pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	n := len(seeds) / c.sk
	if len(seeds) != n*c.sk || len(enc) != n*c.pk || len(ss) != n*c.ss || (ok != nil && len(ok) != n) {
		panic("cb200: " + c.name + "Encaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	pr, prs := hpkeKey(pkR, n, c.pk, c.name+"Encaps")
	status := make([]byte, n)
	err := call(func() C.int {
		if skS == nil {
			switch c.id {
			case HPKEP384HKDFSHA384:
				return C.cb200_hpke_p384_encaps(pr, prs, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
			case HPKEP521HKDFSHA512:
				return C.cb200_hpke_p521_encaps(pr, prs, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
			}
			return C.cb200_hpke_p256_encaps(pr, prs, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
		}
		sp, sps := hpkeKey(skS, n, c.sk, c.name+"Encaps")
		switch c.id {
		case HPKEP384HKDFSHA384:
			return C.cb200_hpke_p384_auth_encaps(pr, prs, sp, sps, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
		case HPKEP521HKDFSHA512:
			return C.cb200_hpke_p521_auth_encaps(pr, prs, sp, sps, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
		}
		return C.cb200_hpke_p256_auth_encaps(pr, prs, sp, sps, u8(seeds), u8(enc), u8(ss), u8(status), C.size_t(n))
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

func (c nist) decaps(skR, enc, pkS, ss []byte, ok []bool) error {
	n := len(enc) / c.pk
	if len(enc) != n*c.pk || len(ss) != n*c.ss || (ok != nil && len(ok) != n) {
		panic("cb200: " + c.name + "Decaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	sr, srs := hpkeKey(skR, n, c.sk, c.name+"Decaps")
	status := make([]byte, n)
	err := call(func() C.int {
		if pkS == nil {
			switch c.id {
			case HPKEP384HKDFSHA384:
				return C.cb200_hpke_p384_decaps(sr, srs, u8(enc), u8(ss), u8(status), C.size_t(n))
			case HPKEP521HKDFSHA512:
				return C.cb200_hpke_p521_decaps(sr, srs, u8(enc), u8(ss), u8(status), C.size_t(n))
			}
			return C.cb200_hpke_p256_decaps(sr, srs, u8(enc), u8(ss), u8(status), C.size_t(n))
		}
		pp, pps := hpkeKey(pkS, n, c.pk, c.name+"Decaps")
		switch c.id {
		case HPKEP384HKDFSHA384:
			return C.cb200_hpke_p384_auth_decaps(sr, srs, u8(enc), pp, pps, u8(ss), u8(status), C.size_t(n))
		case HPKEP521HKDFSHA512:
			return C.cb200_hpke_p521_auth_decaps(sr, srs, u8(enc), pp, pps, u8(ss), u8(status), C.size_t(n))
		}
		return C.cb200_hpke_p256_auth_decaps(sr, srs, u8(enc), pp, pps, u8(ss), u8(status), C.size_t(n))
	})
	for i := range ok {
		ok[i] = status[i] == 0
	}
	return err
}

// HPKEP256Keygen: batched DeriveKeyPair (shortkem.go:63-90) on n seeds of 32 bytes; pk: n*65, sk: n*32.
func HPKEP256Keygen(seeds, pk, sk []byte) error { return nistP256.keygen(seeds, pk, sk) }

// HPKEP256Encaps: batched Encap, or AuthEncap when skS is not nil.  pkR (65 bytes) and skS (32): one key or n keys
// each; seeds: n*32; enc: n*65; ss: n*32.  After the whole batch ran, ErrPrivKey (hpke.ErrInvalidKEMPrivateKey for the
// caller) is returned if any skS is not in [1, n - 1], else ErrPubKey (hpke.ErrInvalidKEMPublicKey) if any pkR is not
// a P-256 point; ok[i] (may be nil) tells which operations failed.
func HPKEP256Encaps(pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	return nistP256.encaps(pkR, skS, seeds, enc, ss, ok)
}

// HPKEP256Decaps: batched Decap, or AuthDecap when pkS is not nil.  skR (32 bytes) and pkS (65): one key or n keys
// each; enc: n*65; ss: n*32.  Errors as HPKEP256Encaps (an invalid skR is ErrPrivKey, an invalid enc or pkS ErrPubKey).
func HPKEP256Decaps(skR, enc, pkS, ss []byte, ok []bool) error { return nistP256.decaps(skR, enc, pkS, ss, ok) }

// HPKEP384Keygen, HPKEP384Encaps, HPKEP384Decaps: the P-256 functions above for DHKEM(P-384, HKDF-SHA384), with
// sk and seeds of 48 bytes, pk and enc of 97 and ss of 48.
func HPKEP384Keygen(seeds, pk, sk []byte) error { return nistP384.keygen(seeds, pk, sk) }
func HPKEP384Encaps(pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	return nistP384.encaps(pkR, skS, seeds, enc, ss, ok)
}
func HPKEP384Decaps(skR, enc, pkS, ss []byte, ok []bool) error { return nistP384.decaps(skR, enc, pkS, ss, ok) }

// HPKEP521Keygen, HPKEP521Encaps, HPKEP521Decaps: the same for DHKEM(P-521, HKDF-SHA512), with sk and seeds of 66
// bytes, pk and enc of 133 and ss of 64.
func HPKEP521Keygen(seeds, pk, sk []byte) error { return nistP521.keygen(seeds, pk, sk) }
func HPKEP521Encaps(pkR, skS, seeds, enc, ss []byte, ok []bool) error {
	return nistP521.encaps(pkR, skS, seeds, enc, ss, ok)
}
func HPKEP521Decaps(skR, enc, pkS, ss []byte, ok []bool) error { return nistP521.decaps(skR, enc, pkS, ss, ok) }

// FrodoKEM-640-SHAKE sizes (kem/frodo/frodo640shake/frodo.go:32-51).
const (
	Frodo640SHAKEPublicKeySize         = 9616
	Frodo640SHAKEPrivateKeySize        = 19888
	Frodo640SHAKECiphertextSize        = 9720
	Frodo640SHAKESharedKeySize         = 16
	Frodo640SHAKESeedSize              = 48
	Frodo640SHAKEEncapsulationSeedSize = 16
)

// Frodo640SHAKEKeygen: batched DeriveKeyPair (frodo.go:84-135) on n seeds of 48 bytes; pk: n*9616, sk: n*19888.
func Frodo640SHAKEKeygen(seeds, pk, sk []byte) error {
	n := len(seeds) / Frodo640SHAKESeedSize
	if len(seeds) != n*Frodo640SHAKESeedSize || len(pk) != n*Frodo640SHAKEPublicKeySize ||
		len(sk) != n*Frodo640SHAKEPrivateKeySize {
		panic("cb200: Frodo640SHAKEKeygen buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int { return C.cb200_frodo640shake_keygen(u8(seeds), u8(pk), u8(sk), C.size_t(n)) })
}

// Frodo640SHAKEEncaps: batched EncapsulateDeterministically (frodo.go:160-240).  pk: one packed key (shared by the
// batch: A and H(pk) are computed once and S'A runs as one tensor-core GEMM) or n keys; seeds: n*16 bytes; ct: n*9720;
// ss: n*16.  FrodoKEM has no failing inputs.
func Frodo640SHAKEEncaps(pk, seeds, ct, ss []byte) error {
	n := len(seeds) / Frodo640SHAKEEncapsulationSeedSize
	if len(seeds) != n*Frodo640SHAKEEncapsulationSeedSize || len(ct) != n*Frodo640SHAKECiphertextSize ||
		len(ss) != n*Frodo640SHAKESharedKeySize {
		panic("cb200: Frodo640SHAKEEncaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	p, ps := hpkeKey(pk, n, Frodo640SHAKEPublicKeySize, "Frodo640SHAKEEncaps")
	return call(func() C.int { return C.cb200_frodo640shake_encaps(p, ps, u8(seeds), u8(ct), u8(ss), C.size_t(n)) })
}

// Frodo640SHAKEDecaps: batched Decapsulate (frodo.go:247-329).  sk: one packed key (shared by the batch) or n keys;
// ct: n*9720 bytes; ss: n*16.  Never fails: a ciphertext that does not re-encrypt gives F(ct || s).
func Frodo640SHAKEDecaps(sk, ct, ss []byte) error {
	n := len(ct) / Frodo640SHAKECiphertextSize
	if len(ct) != n*Frodo640SHAKECiphertextSize || len(ss) != n*Frodo640SHAKESharedKeySize {
		panic("cb200: Frodo640SHAKEDecaps buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	k, ks := hpkeKey(sk, n, Frodo640SHAKEPrivateKeySize, "Frodo640SHAKEDecaps")
	return call(func() C.int { return C.cb200_frodo640shake_decaps(k, ks, u8(ct), u8(ss), C.size_t(n)) })
}

// PinnedBytes returns a Go slice over cudaHostAlloc'd memory: large batches should live
// here so that host<->device copies run at full PCIe speed and overlap with the kernels.
func PinnedBytes(n int) ([]byte, func()) {
	runtime.LockOSThread()
	p := C.cb200_host_alloc(C.size_t(n))
	if p == nil {
		msg := C.GoString(C.cb200_last_error())
		runtime.UnlockOSThread()
		panic(msg)
	}
	runtime.UnlockOSThread()
	return unsafe.Slice((*byte)(p), n), func() { C.cb200_host_free(p) }
}

// KeccakF1600 permutes every 25-lane state in place: the batched counterpart of (*keccakf1600.StateX4).Permute
// (simd/keccakf1600/f1600x.go:115-121); turbo selects the 12-round variant.
func KeccakF1600(states [][25]uint64, turbo bool) error {
	if len(states) == 0 {
		return nil
	}
	t := C.int(0)
	if turbo {
		t = 1
	}
	return call(func() C.int {
		return C.cb200_keccak_f1600((*C.uint64_t)(unsafe.Pointer(&states[0])), C.size_t(len(states)), t)
	})
}

// KyberDeriveUniform: (*Poly).DeriveUniform (pke/kyber/internal/common/sample.go:192-236) for len(polys) (seed, x, y)
// triples; seeds holds one 32-byte seed (shared) or one per polynomial, xy two bytes per polynomial.
func KyberDeriveUniform(polys [][256]int16, seeds []byte, xy []byte) error {
	n := len(polys)
	if len(xy) != 2*n || (len(seeds) != 32 && len(seeds) != 32*n) {
		panic("cb200: KyberDeriveUniform buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	stride := C.size_t(32)
	if len(seeds) == 32 {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_kyber_derive_uniform((*C.int16_t)(unsafe.Pointer(&polys[0])), (*C.uint8_t)(unsafe.Pointer(&seeds[0])),
			stride, (*C.uint8_t)(unsafe.Pointer(&xy[0])), C.size_t(n))
	})
}

// ---- OPRF servers (RFC 9497, the reference's oprf package) over P-256, P-384 and P-521

// Suite ids of cb200_oprf_* (include/circl_b200.h).
const (
	OPRFP256SHA256 = int(C.CB200_OPRF_P256_SHA256)
	OPRFP384SHA384 = int(C.CB200_OPRF_P384_SHA384)
	OPRFP521SHA512 = int(C.CB200_OPRF_P521_SHA512)
)

// OPRFSizes returns (Ne, Ns, Nh, proof size) of a suite.
func OPRFSizes(suite int) (ne, ns, nh, proof int) {
	s := C.int(suite)
	return int(C.cb200_oprf_element_size(s)), int(C.cb200_oprf_scalar_size(s)), int(C.cb200_oprf_output_size(s)),
		int(C.cb200_oprf_proof_size(s))
}

// oprfSizes is OPRFSizes for a suite the library serves (an unknown suite panics, as a wrong length does)
func oprfSizes(suite int) (ne, ns, nh, proof int) {
	ne, ns, nh, proof = OPRFSizes(suite)
	if ne == 0 {
		panic("cb200: unknown OPRF suite")
	}
	return
}

// oprfKeyLen is the length of the sk argument: one key (shared) or one per op
func oprfKeyLen(ns, n int, shared bool) int {
	if shared {
		return ns
	}
	return n * ns
}

func optPtr(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return u8(b)
}

// OPRFDeriveKey: oprf.DeriveKey (oprf/keys.go:103-132) on n 32-byte seeds with one info; sk receives n*Ns bytes, pk
// n*Ne (compressed).  A buffer of the wrong length or an unknown suite panics.
func OPRFDeriveKey(suite, mode int, seeds, info, sk, pk []byte) error {
	ne, ns, _, _ := oprfSizes(suite)
	n := len(seeds) / 32
	if len(seeds) != n*32 || len(sk) != n*ns || len(pk) != n*ne {
		panic("cb200: OPRFDeriveKey seeds/sk/pk have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_oprf_derive_key(C.int(suite), C.int(mode), u8(seeds), optPtr(info), C.size_t(len(info)), u8(sk),
			u8(pk), C.size_t(n))
	})
}

// OPRFEvaluate: Server / VerifiableServer / PartialObliviousServer.Evaluate (oprf/server.go:23-85) on n requests of
// m blinded elements each (n*m*Ne bytes).  sk holds one key (shared) or n; rnd n*Ns bytes of proof randomness (modes 1
// and 2).  evaluated receives n*m*Ne bytes, proof n*2*Ns (modes 1 and 2), status one byte per request (0 = ok; the
// failed requests' rows are zero).  A buffer of the wrong length, 1 <= m <= 65535 unmet or an unknown suite panics.
func OPRFEvaluate(suite, mode int, sk []byte, shared bool, blinded []byte, m int, rnd, info, evaluated, proof,
	status []byte) error {
	ne, ns, _, np := oprfSizes(suite)
	n := len(status)
	if m < 1 || m > 65535 || len(sk) != oprfKeyLen(ns, n, shared) || len(blinded) != n*m*ne ||
		len(evaluated) != n*m*ne || (mode != 0 && (len(rnd) != n*ns || len(proof) != n*np)) {
		panic("cb200: OPRFEvaluate buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	stride := C.size_t(ns)
	if shared {
		stride = 0
	}
	var rp, pp *C.uint8_t // mode 0 reads no randomness and writes no proof
	if mode != 0 {
		rp, pp = u8(rnd), u8(proof)
	}
	return call(func() C.int {
		return C.cb200_oprf_evaluate(C.int(suite), C.int(mode), u8(sk), stride, u8(blinded), C.size_t(m), rp,
			optPtr(info), C.size_t(len(info)), u8(evaluated), pp, u8(status), C.size_t(n))
	})
}

// OPRFFullEvaluate: the servers' FullEvaluate (oprf/server.go:97-117) on len(inputs) inputs of at most 65535 bytes;
// sk holds Ns bytes (shared) or len(inputs)*Ns; out receives len(inputs)*Nh bytes, status one byte per op.  A buffer of
// the wrong length or an unknown suite panics.
func OPRFFullEvaluate(suite, mode int, sk []byte, shared bool, inputs [][]byte, info, out, status []byte) error {
	_, ns, nh, _ := oprfSizes(suite)
	n := len(inputs)
	if len(sk) != oprfKeyLen(ns, n, shared) || len(out) != n*nh || len(status) != n {
		panic("cb200: OPRFFullEvaluate buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(inputs)
	stride := C.size_t(ns)
	if shared {
		stride = 0
	}
	return call(func() C.int {
		return C.cb200_oprf_full_evaluate(C.int(suite), C.int(mode), u8(sk), stride, u8(blob),
			(*C.uint64_t)(unsafe.Pointer(&off[0])), optPtr(info), C.size_t(len(info)), u8(out), u8(status), C.size_t(n))
	})
}

// ---- RSA blind signatures (RFC 9474, RSABSSA-SHA384, the reference's blindsign/blindrsa package), server side
// Keys are big-endian byte strings, one key per call; rows are kLen = BRSAModulusBytes(N) bytes.

// Variant ids, in the reference's blindrsa.Variant order.
const (
	BRSASHA384PSSRandomized        = int(C.CB200_BRSA_SHA384_PSS_RANDOMIZED)
	BRSASHA384PSSZeroRandomized    = int(C.CB200_BRSA_SHA384_PSSZERO_RANDOMIZED)
	BRSASHA384PSSDeterministic     = int(C.CB200_BRSA_SHA384_PSS_DETERMINISTIC)
	BRSASHA384PSSZeroDeterministic = int(C.CB200_BRSA_SHA384_PSSZERO_DETERMINISTIC)
)

// BRSAModulusBytes returns kLen of the modulus N, or 0 outside 2048 to 4096 bits.
func BRSAModulusBytes(N []byte) int {
	if len(N) == 0 {
		return 0
	}
	return int(C.cb200_brsa_modulus_bytes(u8(N), C.size_t(len(N))))
}

// BRSABlindSign: Signer.BlindSign (blindsign/blindrsa/brsa.go:237-257) on n blinded rows of kLen under the CRT key
// (N, e, p, q, dp, dq, qinv); sig receives n*kLen bytes, status n bytes (1 = c > N, 2 = the s^e mod N == c check
// failed; that row is zero).  A buffer of the wrong length panics; a key outside the served range is an error.
func BRSABlindSign(N, e, p, q, dp, dq, qinv, blinded, sig, status []byte) error {
	k := BRSAModulusBytes(N)
	n := len(status)
	if k == 0 || len(blinded) != n*k || len(sig) != n*k {
		panic("cb200: BRSABlindSign buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	for _, f := range [][]byte{e, p, q, dp, dq, qinv} {
		if len(f) == 0 {
			panic("cb200: BRSABlindSign key field is empty")
		}
	}
	return call(func() C.int {
		return C.cb200_brsa_blind_sign(u8(N), C.size_t(len(N)), u8(e), C.size_t(len(e)), u8(p), C.size_t(len(p)),
			u8(q), C.size_t(len(q)), u8(dp), C.size_t(len(dp)), u8(dq), C.size_t(len(dq)), u8(qinv),
			C.size_t(len(qinv)), u8(blinded), u8(sig), u8(status), C.size_t(n))
	})
}

// BRSAVerify: Verifier.Verify (brsa.go:214) of msgs[i] and the kLen-byte sigs row i under (N, e) for a variant;
// status receives n bytes (0 valid, 1 = s >= N, 2 = an inconsistent encoding; both rsa.ErrVerification).
func BRSAVerify(variant int, N, e []byte, msgs [][]byte, sigs, status []byte) error {
	k := BRSAModulusBytes(N)
	n := len(msgs)
	if k == 0 || len(e) == 0 || len(sigs) != n*k || len(status) != n {
		panic("cb200: BRSAVerify buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	return call(func() C.int {
		return C.cb200_brsa_verify(C.int(variant), u8(N), C.size_t(len(N)), u8(e), C.size_t(len(e)), u8(blob),
			(*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sigs), u8(status), C.size_t(n))
	})
}

// ---- Partially blind RSA signatures (RSAPBSSA-SHA384, the reference's blindsign/blindrsa/partiallyblindrsa
// package), server side.  Keys are big-endian byte strings, one key per call; rows are kLen = BRSAModulusBytes(N)
// bytes; each op has its own metadata, which selects the key it is signed and verified under.

// PBRSACheckKey is NewSigner's safe-prime test (pbrsa.go:324-343) on the host: an error unless (p - 1) / 2 and
// (q - 1) / 2 pass 20 Miller-Rabin rounds and the key is in the served range.  It needs no device.
func PBRSACheckKey(N, p, q []byte) error {
	if len(N) == 0 || len(p) == 0 || len(q) == 0 {
		panic("cb200: PBRSACheckKey key field is empty")
	}
	return call(func() C.int {
		return C.cb200_pbrsa_check_key(u8(N), C.size_t(len(N)), u8(p), C.size_t(len(p)), u8(q), C.size_t(len(q)))
	})
}

// PBRSABlindSign: Signer.BlindSign (pbrsa.go:350-375) on n blinded rows of kLen, op i under metadata[i], with the key
// (N, p, q, qinv = q^-1 mod p); sig receives n*kLen bytes, status n bytes (1 = c > N, 2 = the s^e' mod N == c check
// failed; that row is zero).  A buffer of the wrong length panics; a key outside the served range is an error.
func PBRSABlindSign(N, p, q, qinv, blinded []byte, metadata [][]byte, sig, status []byte) error {
	k := BRSAModulusBytes(N)
	n := len(status)
	if k == 0 || len(blinded) != n*k || len(sig) != n*k || len(metadata) != n {
		panic("cb200: PBRSABlindSign buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	for _, f := range [][]byte{p, q, qinv} {
		if len(f) == 0 {
			panic("cb200: PBRSABlindSign key field is empty")
		}
	}
	blob, off := packMsgs(metadata)
	return call(func() C.int {
		return C.cb200_pbrsa_blind_sign(u8(N), C.size_t(len(N)), u8(p), C.size_t(len(p)), u8(q), C.size_t(len(q)),
			u8(qinv), C.size_t(len(qinv)), u8(blinded), u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])), u8(sig),
			u8(status), C.size_t(n))
	})
}

// PBRSAVerify: Verifier.Verify (pbrsa.go:244-251) of msgs[i] under metadata[i] and the kLen-byte sigs row i under N;
// status receives n bytes (0 valid, 1 = s >= N, 2 = an inconsistent encoding; both rsa.ErrVerification).
func PBRSAVerify(N []byte, msgs, metadata [][]byte, sigs, status []byte) error {
	k := BRSAModulusBytes(N)
	n := len(msgs)
	if k == 0 || len(metadata) != n || len(sigs) != n*k || len(status) != n {
		panic("cb200: PBRSAVerify buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	blob, off := packMsgs(msgs)
	mblob, moff := packMsgs(metadata)
	return call(func() C.int {
		return C.cb200_pbrsa_verify(u8(N), C.size_t(len(N)), u8(blob), (*C.uint64_t)(unsafe.Pointer(&off[0])),
			u8(mblob), (*C.uint64_t)(unsafe.Pointer(&moff[0])), u8(sigs), u8(status), C.size_t(n))
	})
}

// Prio3Config describes one Prio3 instance (draft-irtf-cfrg-vdaf-14, the reference's vdaf/prio3): Kind is the
// reference's algorithm ID (1 Count, 2 Sum, 3 SumVec, 4 Histogram, 5 MultiHotCountVec); only the parameters of that
// kind are read.
type Prio3Config struct {
	Kind, NumShares                                     uint32
	MaxMeasurement, Length, Bits, ChunkLength, MaxWeight uint64
	Context                                             []byte
}

// Prio3Sizes are the wire sizes of one instance (cb200_prio3_get_sizes).
type Prio3Sizes struct {
	InputShareLeader, InputShareHelper, PublicShare, PrepShare, PrepMsg, PrepState, OutShare, AggShare int
}

// cfgOf returns the C configuration; the context is copied to C memory by the caller's pinning rules (cgo allows Go
// memory that holds no Go pointers to be passed for the duration of the call).
func cfgOf(c *Prio3Config) C.cb200_prio3_config {
	var k C.cb200_prio3_config
	k.kind, k.num_shares = C.uint32_t(c.Kind), C.uint32_t(c.NumShares)
	k.max_measurement, k.length, k.bits = C.uint64_t(c.MaxMeasurement), C.uint64_t(c.Length), C.uint64_t(c.Bits)
	k.chunk_length, k.max_weight = C.uint64_t(c.ChunkLength), C.uint64_t(c.MaxWeight)
	k.context_len = C.size_t(len(c.Context))
	return k
}

func u8opt(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return u8(b)
}

// prio3Call runs f with the configuration whose context points at a C copy of c.Context.
func prio3Call(c *Prio3Config, f func(k *C.cb200_prio3_config) C.int) error {
	k := cfgOf(c)
	if len(c.Context) > 0 {
		p := C.CBytes(c.Context)
		defer C.free(p)
		k.context = (*C.uint8_t)(p)
	}
	return call(func() C.int { return f(&k) })
}

// Prio3GetSizes validates the configuration as the reference's New does (an error otherwise) and returns its sizes.
// It needs no device.
func Prio3GetSizes(c *Prio3Config) (Prio3Sizes, error) {
	var z C.cb200_prio3_sizes
	err := prio3Call(c, func(k *C.cb200_prio3_config) C.int { return C.cb200_prio3_get_sizes(k, &z) })
	return Prio3Sizes{int(z.input_share_leader), int(z.input_share_helper), int(z.public_share), int(z.prep_share),
		int(z.prep_msg), int(z.prep_state), int(z.out_share), int(z.agg_share)}, err
}

// Prio3PrepInit: PrepInit (prio3.go:245-324) of len(status) reports under one verify key as aggregator aggID; rows
// back to back in the reference's encodings.  status: 1 an element >= p, 2 ErrJointRand, 4 ErrInvalidEval; failed
// rows are zero.  Buffers of the wrong length panic.
func Prio3PrepInit(c *Prio3Config, z Prio3Sizes, verifyKey []byte, aggID uint8, nonces, publicShares, inputShares,
	prepStates, prepShares, status []byte) error {
	n := len(status)
	in := z.InputShareLeader
	if aggID != 0 {
		in = z.InputShareHelper
	}
	if len(verifyKey) != 32 || len(nonces) != 16*n || len(publicShares) != z.PublicShare*n ||
		len(inputShares) != in*n || len(prepStates) != z.PrepState*n || len(prepShares) != z.PrepShare*n {
		panic("cb200: Prio3PrepInit buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return prio3Call(c, func(k *C.cb200_prio3_config) C.int {
		return C.cb200_prio3_prep_init(k, u8(verifyKey), C.uint32_t(aggID), u8(nonces), u8opt(publicShares),
			u8(inputShares), u8(prepStates), u8(prepShares), u8(status), C.size_t(n))
	})
}

// Prio3PrepSharesToPrep: PrepSharesToPrep (:332-377); row i of prepShares is the NumShares prep shares of report i.
// status: 1 an element >= p, 8 ErrProofVerify.
func Prio3PrepSharesToPrep(c *Prio3Config, z Prio3Sizes, prepShares, prepMsgs, status []byte) error {
	n := len(status)
	if len(prepShares) != int(c.NumShares)*z.PrepShare*n || len(prepMsgs) != z.PrepMsg*n {
		panic("cb200: Prio3PrepSharesToPrep buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return prio3Call(c, func(k *C.cb200_prio3_config) C.int {
		return C.cb200_prio3_prep_shares_to_prep(k, u8(prepShares), u8opt(prepMsgs), u8(status), C.size_t(n))
	})
}

// Prio3PrepNext: PrepNext (:386-403).  status: 2 ErrJointRand.
func Prio3PrepNext(c *Prio3Config, z Prio3Sizes, prepStates, prepMsgs, outShares, status []byte) error {
	n := len(status)
	if len(prepStates) != z.PrepState*n || len(prepMsgs) != z.PrepMsg*n || len(outShares) != z.OutShare*n {
		panic("cb200: Prio3PrepNext buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return prio3Call(c, func(k *C.cb200_prio3_config) C.int {
		return C.cb200_prio3_prep_next(k, u8(prepStates), u8opt(prepMsgs), u8(outShares), u8(status), C.size_t(n))
	})
}

// Prio3Aggregate: AggregateInit + AggregateUpdate (:408-420) of the out shares whose status byte is 0 (all of them
// for a nil status) into aggShare.
func Prio3Aggregate(c *Prio3Config, z Prio3Sizes, outShares, status, aggShare []byte) error {
	n := len(outShares) / max(z.OutShare, 1)
	if len(outShares) != z.OutShare*n || (status != nil && len(status) != n) || len(aggShare) != z.AggShare {
		panic("cb200: Prio3Aggregate buffers have the wrong length")
	}
	if n == 0 {
		clear(aggShare)
		return nil
	}
	return prio3Call(c, func(k *C.cb200_prio3_config) C.int {
		return C.cb200_prio3_aggregate(k, u8opt(outShares), u8opt(status), u8(aggShare), C.size_t(n))
	})
}

// ---- Threshold RSA (the reference's tss/rsa, Shoup's protocol 1).  N and e are big-endian byte strings; rows are
// kLen = BRSAModulusBytes(N) bytes back to back.  Served: 2 <= players <= 64, threshold <= k <= 64, u16 indices.

// TSSRSASignShare: KeyShare.Sign (keyshare.go:188-256) of n digests (n rows of kLen) with the exponent E = 2 Delta s_i
// (or the share's cached twoDeltaSi); xi receives the n shares.
func TSSRSASignShare(N []byte, players int, E, digests, xi []byte) error {
	k := BRSAModulusBytes(N)
	n := 0
	if k != 0 {
		n = len(digests) / k
	}
	if k == 0 || len(E) == 0 || len(digests) != n*k || len(xi) != n*k {
		panic("cb200: TSSRSASignShare buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_tssrsa_sign_share(u8(N), C.size_t(len(N)), C.int(players), u8(E), C.size_t(len(E)),
			u8(digests), u8(xi), C.size_t(n))
	})
}

// TSSRSACombine: CombineSignShares (rsa_threshold.go:207-293) of n ops after the share parameter checks: op i combines
// the k shares xi row i (k kLen bytes) of the indices idx[i*k:(i+1)*k] for the padded message msgs row i; sig receives
// n rows, status n bytes (0, 1 = ErrInvalidCalc, 2 = "rsa: internal error"; failed rows zero).
func TSSRSACombine(N, e []byte, players, threshold, k int, idx []uint16, xi, msgs, sig, status []byte) error {
	kl := BRSAModulusBytes(N)
	n := len(status)
	if kl == 0 || len(e) == 0 || k < 1 || len(idx) != n*k || len(xi) != n*k*kl || len(msgs) != n*kl ||
		len(sig) != n*kl {
		panic("cb200: TSSRSACombine buffers have the wrong length")
	}
	if n == 0 {
		return nil
	}
	return call(func() C.int {
		return C.cb200_tssrsa_combine(u8(N), C.size_t(len(N)), u8(e), C.size_t(len(e)), C.int(players),
			C.int(threshold), C.int(k), (*C.uint16_t)(unsafe.Pointer(&idx[0])), u8(xi), u8(msgs), u8(sig), u8(status),
			C.size_t(n))
	})
}
