// RSA blind signatures (RFC 9474, RSABSSA-SHA384), server side: BlindSign under one private key and Verify under one
// public key per call, batched on the device with one thread per operation.  The arithmetic is rsa.cuh:
//   BlindSign   brsa_sign_kernel<WP, WN>    c^dp mod p and c^dq mod q at WP words, Garner, s^e mod N == c at WN words
//   Verify      brsa_verify_kernel<WN>      s^e mod N, SHA-384 of the message, EMSA-PSS decode
// WP is 32, 48 or 64 words by the larger prime, WN 64, 96 or 128 by N.  The key's Montgomery constants are computed
// on the host once per call and copied into the call's level-1 work area; every thread reads the same key words.
// Like the reference, the library does not wipe key material: the host copies and the work area keep the CRT key
// until they are reused.
// Timed under the profiling class rsa.
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "rsa.cuh"
#include "rsa_host.h"

namespace cb200 {
namespace brsak {

template <int WP, int WN>
__global__ void __launch_bounds__(128) brsa_sign_kernel(const rsa::SignKey<WP, WN>* __restrict__ K,
                                                        const uint8_t* __restrict__ in, size_t in_stride,
                                                        uint8_t* __restrict__ out, size_t out_stride,
                                                        uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  status[i] = (uint8_t)rsa::blind_sign<WP, WN>(out + i * out_stride, in + i * in_stride, *K);
}

template <int WN>
__global__ void __launch_bounds__(128) brsa_verify_kernel(const rsa::VerifyKey<WN>* __restrict__ K,
                                                          const uint8_t* __restrict__ msgs,
                                                          const uint64_t* __restrict__ msg_off,
                                                          const uint8_t* __restrict__ sig, size_t sig_stride,
                                                          uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t m0 = msg_off[i], m1 = msg_off[i + 1];
  // a message of 2^31 bytes or more, or offsets that decrease (only a device-pointer call can pass either), fails its
  // op rather than being hashed with a truncated length
  status[i] = m1 < m0 || m1 - m0 > 0x7fffffff ? 2 : (uint8_t)rsa::verify<WN>(msgs + m0, m1 - m0, sig + i * sig_stride, *K);
}

// ---------------------------------------------------------------- host side
using namespace rsah;

struct PubKey {
  Modulus m;
  uint32_t e;
};
// N of 2048 to 4096 bits and an odd e with 3 <= e < 2^32
static int parse_public(const char* fn, const uint8_t* N, size_t N_len, const uint8_t* e, size_t e_len, PubKey* k) {
  if (!N || !e) {
    set_error("%s: null key field", fn);
    return CB200_ERR_ARG;
  }
  int rc = parse_modulus(fn, N, N_len, &k->m);
  if (rc) return rc;
  const Words ew = be_words(e, e_len);
  if (ew.size() != 1 || ew[0] < 3 || !(ew[0] & 1)) {
    set_error("%s: the public exponent must be odd, at least 3 and below 2^32", fn);
    return CB200_ERR_ARG;
  }
  k->e = ew[0];
  return 0;
}

struct PrivKey {
  PubKey pub;
  Words p, q, dp, dq, qinv;
  int wp;
};
static int parse_private(const char* fn, const uint8_t* const* f, const size_t* len, PrivKey* k) {
  int rc = parse_public(fn, f[0], len[0], f[1], len[1], &k->pub);
  if (rc) return rc;
  for (int i = 2; i < 7; i++)
    if (!f[i]) {
      set_error("%s: null key field", fn);
      return CB200_ERR_ARG;
    }
  rc = parse_primes(fn, k->pub.m.n, f[2], len[2], f[3], len[3], &k->p, &k->q, &k->wp);
  if (rc) return rc;
  k->dp = be_words(f[4], len[4]);
  k->dq = be_words(f[5], len[5]);
  k->qinv = be_words(f[6], len[6]);
  if ((int)std::max({k->dp.size(), k->dq.size(), k->qinv.size()}) > k->wp) {
    set_error("%s: dp, dq and qinv must be reduced mod p - 1, q - 1 and p", fn);
    return CB200_ERR_ARG;
  }
  return 0;
}

// the sign body at one pair of word counts: key constants once per call, then the batch
template <int WP, int WN>
static int sign(const char* fn, const PrivKey& k, const uint8_t* blinded, uint8_t* sig, uint8_t* status, size_t n) {
  rsa::SignKey<WP, WN> K;
  load_crt<WP, WN>(K, k.pub.m, k.p, k.q, k.qinv);
  fill(K.dp, WP, k.dp);
  fill(K.dq, WP, k.dq);
  K.e = k.pub.e;
  const size_t kl = (size_t)K.klen;
  Batch b{fn, n, sig, 1u << 14, 1u << 10, {{blinded, kl, kl, kIn}, {sig, kl, kl, kOut}, {status, 1, 1, kStatus}}, {}};
  return run_keyed(b, K, [&](const rsa::SignKey<WP, WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    brsa_sign_kernel<WP, WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r[0].p, r[0].stride, r[1].p, r[1].stride, r[2].p,
                                                               cnt);
  });
}

template <int WN>
static int verify(const char* fn, const PubKey& k, int slen, const uint8_t* msgs, const uint64_t* msg_off,
                  const uint8_t* sigs, uint8_t* status, size_t n) {
  rsa::VerifyKey<WN> K;
  load_mod<WN>(K.n, k.m.n);
  K.e = k.e;
  K.klen = k.m.klen;
  K.slen = slen;
  const size_t kl = (size_t)K.klen;
  Batch b{fn, n, sigs, 1u << 14, 1u << 10, {{sigs, kl, kl, kIn}, {status, 1, 1, kStatus}},
          {{!aligned({msg_off}, {}, 8), "%s: device msg_off must be 8-byte aligned"}}, msgs, msg_off};
  return run_keyed(b, K, [&](const rsa::VerifyKey<WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    brsa_verify_kernel<WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r.msgs, r.msg_off, r[0].p, r[0].stride, r[1].p, cnt);
  });
}

}  // namespace brsak
}  // namespace cb200

using namespace cb200;
using namespace cb200::brsak;

extern "C" {

size_t cb200_brsa_modulus_bytes(const uint8_t* N, size_t N_len) {
  if (!N) return 0;
  const int bits = bitlen(be_words(N, N_len));
  return bits >= 2048 && bits <= 4096 ? (size_t)(bits + 7) / 8 : 0;
}

int cb200_brsa_blind_sign(const uint8_t* N, size_t N_len, const uint8_t* e, size_t e_len, const uint8_t* p,
                          size_t p_len, const uint8_t* q, size_t q_len, const uint8_t* dp, size_t dp_len,
                          const uint8_t* dq, size_t dq_len, const uint8_t* qinv, size_t qinv_len,
                          const uint8_t* blinded, uint8_t* sig, uint8_t* status, size_t n) {
  const char* fn = "cb200_brsa_blind_sign";
  const uint8_t* f[7] = {N, e, p, q, dp, dq, qinv};
  const size_t len[7] = {N_len, e_len, p_len, q_len, dp_len, dq_len, qinv_len};
  PrivKey k;
  int rc = parse_private(fn, f, len, &k);
  if (rc) return rc;
  if (!blinded || !sig || !status) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  return with_words(k.wp, k.pub.m.wn, [&](auto wp, auto wn) { return sign<wp, wn>(fn, k, blinded, sig, status, n); });
}

int cb200_brsa_verify(int variant, const uint8_t* N, size_t N_len, const uint8_t* e, size_t e_len,
                      const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* sigs, uint8_t* status, size_t n) {
  const char* fn = "cb200_brsa_verify";
  if (variant < CB200_BRSA_SHA384_PSS_RANDOMIZED || variant > CB200_BRSA_SHA384_PSSZERO_DETERMINISTIC) {
    set_error("%s: unknown variant %d", fn, variant);
    return CB200_ERR_ARG;
  }
  PubKey k;
  int rc = parse_public(fn, N, N_len, e, e_len, &k);
  if (rc) return rc;
  if (!msgs || !msg_off || !sigs || !status) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!is_device_ptr(msg_off))
    for (size_t i = 0; i < n; i++)
      if (msg_off[i + 1] < msg_off[i] || msg_off[i + 1] - msg_off[i] > 0x7fffffff) {
        set_error("%s: message %zu has a bad offset or is 2^31 bytes or longer", fn, i);
        return CB200_ERR_ARG;
      }
  const int slen = (variant == CB200_BRSA_SHA384_PSS_RANDOMIZED || variant == CB200_BRSA_SHA384_PSS_DETERMINISTIC)
                       ? rsa::kHash
                       : 0;
  return with_words(k.m.wn, [&](auto wn) { return verify<wn>(fn, k, slen, msgs, msg_off, sigs, status, n); });
}

}  // extern "C"
