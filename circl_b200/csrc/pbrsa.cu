// Partially blind RSA signatures (draft-amjad-cfrg-partially-blind-rsa, RSAPBSSA-SHA384), server side: BlindSign under
// one private key and Verify under one public key per call, each op with its own metadata, batched on the device with
// one thread per operation.  The arithmetic is rsa.cuh:
//   BlindSign   pbrsa_sign_kernel<WP, WN>   e' from the metadata, d'_p and d'_q by Fermat inversion mod p' and q',
//                                           c^d'_p mod p and c^d'_q mod q, Garner, s^e' mod N == c at WN words
//   Verify      pbrsa_verify_kernel<WN>     e' from the metadata, s^e' mod N, SHA-384 of the framed message, EMSA-PSS
// WP is 32, 48 or 64 words by the larger prime, WN 64, 96 or 128 by N, as in brsa.cu.  The key's Montgomery constants
// (for p, q, p', q' and N) and the pad states of HKDF's salt are computed on the host once per call and copied into the
// call's level-1 work area.  The safe-prime test of the key (cb200_pbrsa_check_key) is the caller's, once per key.
// Timed under the profiling class rsa.
#include <random>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "rsa.cuh"
#include "rsa_host.h"

namespace cb200 {
namespace pbrsak {

// metadata of at most kMaxMeta bytes, and framed Verify messages ("msg" || I2OSP(len(meta), 4) || meta || msg) below
// 2^31 bytes: the hash lengths then fit an int
constexpr uint64_t kMaxMeta = 0x7fffffff - 7;
__host__ __device__ inline bool bad_lengths(uint64_t ml, uint64_t len) { return ml > kMaxMeta || len > kMaxMeta - ml; }

template <int WP, int WN>
__global__ void __launch_bounds__(128) pbrsa_sign_kernel(const rsa::PbSignKey<WP, WN>* __restrict__ K,
                                                         const uint8_t* __restrict__ in, size_t in_stride,
                                                         const uint8_t* __restrict__ meta,
                                                         const uint64_t* __restrict__ meta_off,
                                                         uint8_t* __restrict__ out, size_t out_stride,
                                                         uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t m0 = meta_off[i], m1 = meta_off[i + 1];
  uint8_t* o = out + i * out_stride;
  // offsets that decrease or over-long metadata (only a device-pointer call can pass either) fail the op
  if (m1 < m0 || bad_lengths(m1 - m0, 0)) {
    for (int k = 0; k < K->klen; k++) o[k] = 0;
    status[i] = 2;
    return;
  }
  status[i] = (uint8_t)rsa::pb_blind_sign<WP, WN>(o, in + i * in_stride, meta + m0, (int)(m1 - m0), *K);
}

// Message i is msgs[msg_off[i] .. msg_off[i + 1]).  With mlen (host-pointer calls, staged as one string per op) its
// first mlen[i] bytes are the metadata; else the metadata is meta[meta_off[i] .. meta_off[i + 1]).
template <int WN>
__global__ void __launch_bounds__(128) pbrsa_verify_kernel(const rsa::PbVerifyKey<WN>* __restrict__ K,
                                                           const uint8_t* __restrict__ msgs,
                                                           const uint64_t* __restrict__ msg_off,
                                                           const uint8_t* __restrict__ meta,
                                                           const uint64_t* __restrict__ meta_off,
                                                           const uint64_t* __restrict__ mlen,
                                                           const uint8_t* __restrict__ sig, size_t sig_stride,
                                                           uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t a0 = msg_off[i], a1 = msg_off[i + 1];
  const uint8_t *mp, *gp;
  uint64_t ml, gl;
  bool bad = a1 < a0;
  if (mlen) {
    ml = mlen[i];
    mp = msgs + a0;
    gp = mp + ml;
    gl = a1 - a0 - ml;
  } else {
    const uint64_t b0 = meta_off[i], b1 = meta_off[i + 1];
    bad = bad || b1 < b0;
    ml = b1 - b0;
    mp = meta + b0;
    gp = msgs + a0;
    gl = a1 - a0;
  }
  status[i] = bad || bad_lengths(ml, gl) ? 2 : (uint8_t)rsa::pb_verify<WN>(gp, (int)gl, mp, (int)ml, sig + i * sig_stride, *K);
}

// ---------------------------------------------------------------- host side
using namespace rsah;

struct Key {
  Modulus m;
  Words p, q, qinv;
  int wp;
};
// N, p, q (and qinv when wanted): the brsa key rules, both primes = 3 mod 4 and at least 7 (so p' and q' are odd and
// above 1), qinv < p
static int parse_key(const char* fn, const uint8_t* N, size_t N_len, const uint8_t* p, size_t p_len, const uint8_t* q,
                     size_t q_len, const uint8_t* qinv, size_t qinv_len, bool want_qinv, Key* k) {
  if (!N || !p || !q || (want_qinv && !qinv)) {
    set_error("%s: null key field", fn);
    return CB200_ERR_ARG;
  }
  int rc = parse_modulus(fn, N, N_len, &k->m);
  if (rc) return rc;
  rc = parse_primes(fn, k->m.n, p, p_len, q, q_len, &k->p, &k->q, &k->wp);
  if (rc) return rc;
  if ((k->p[0] & 3) != 3 || (k->q[0] & 3) != 3 || bitlen(k->p) < 3 || bitlen(k->q) < 3) {
    set_error("%s: p and q must be = 3 mod 4 and at least 7, so that (p - 1) / 2 and (q - 1) / 2 are odd", fn);
    return CB200_ERR_ARG;
  }
  if (want_qinv) {
    k->qinv = be_words(qinv, qinv_len);
    if (!less(k->qinv, k->p)) {
      set_error("%s: qinv must be below p", fn);
      return CB200_ERR_ARG;
    }
  }
  return 0;
}

// (x - 1) / 2 and (x - 1) / 2 - 2 of an odd x >= 7
static Words half(const Words& x) {
  Words h(x.size());
  for (size_t j = 0; j < x.size(); j++) h[j] = (x[j] >> 1) | (j + 1 < x.size() ? x[j + 1] << 31 : 0);
  while (!h.empty() && !h.back()) h.pop_back();
  return h;
}
static Words minus2(Words x) {
  uint32_t br = 2;
  for (size_t j = 0; j < x.size() && br; j++) {
    const uint32_t v = x[j];
    x[j] = v - br;
    br = v < br;
  }
  while (!x.empty() && !x.back()) x.pop_back();
  return x;
}

static void salt_states(const Modulus& m, uint64_t (&si)[8], uint64_t (&so)[8]) {
  std::vector<uint8_t> nb(m.klen);
  for (int i = 0; i < m.klen; i++) nb[i] = rsa::be_byte(m.n.data(), m.klen, i);  // n has ceil(klen / 4) words
  rsa::pb_salt_states(si, so, nb.data(), m.klen);
}

template <int WP, int WN>
static int sign(const char* fn, const Key& k, const uint8_t* blinded, const uint8_t* meta, const uint64_t* meta_off,
                uint8_t* sig, uint8_t* status, size_t n) {
  rsa::PbSignKey<WP, WN> K;
  load_crt<WP, WN>(K, k.m, k.p, k.q, k.qinv);
  const Words ph = half(k.p), qh = half(k.q);
  load_mod<WP>(K.ph, ph);
  load_mod<WP>(K.qh, qh);
  fill(K.ph2, WP, minus2(ph));
  fill(K.qh2, WP, minus2(qh));
  salt_states(k.m, K.si, K.so);
  const size_t kl = (size_t)K.klen;
  Batch b{fn, n, sig, 1u << 14, 1u << 10, {{blinded, kl, kl, kIn}, {sig, kl, kl, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({meta_off}, {}, 8), "%s: device meta_off must be 8-byte aligned"}}, meta, meta_off};
  return run_keyed(b, K, [&](const rsa::PbSignKey<WP, WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    pbrsa_sign_kernel<WP, WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r[0].p, r[0].stride, r.msgs, r.msg_off, r[1].p,
                                                                r[1].stride, r[2].p, cnt);
  });
}

// msgs / msg_off: on host-pointer calls the framed strings meta || msg with mlen the metadata lengths; on device-pointer
// calls the caller's messages, with meta / meta_off beside them
template <int WN>
static int verify(const char* fn, const Modulus& m, const uint8_t* msgs, const uint64_t* msg_off, const uint8_t* meta,
                  const uint64_t* meta_off, const uint64_t* mlen, const uint8_t* sigs, uint8_t* status, size_t n) {
  rsa::PbVerifyKey<WN> K;
  load_mod<WN>(K.n, m.n);
  salt_states(m, K.si, K.so);
  K.klen = m.klen;
  const size_t kl = (size_t)m.klen;
  Batch b{fn, n, sigs, 1u << 14, 1u << 10, {{sigs, kl, kl, kIn}, {mlen, 8, 8, kIn}, {status, 1, 1, kStatus}},
          {{!aligned({msg_off, meta_off}, {}, 8), "%s: device msg_off and meta_off must be 8-byte aligned"}}, msgs,
          msg_off};
  return run_keyed(b, K, [&](const rsa::PbVerifyKey<WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    pbrsa_verify_kernel<WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r.msgs, r.msg_off, meta, meta_off,
                                                              (const uint64_t*)r[1].p, r[0].p, r[0].stride, r[2].p, cnt);
  });
}

// offsets of n ops on the host: non-decreasing; false on the first that is not
static bool host_offsets_ok(const uint64_t* off, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (off[i + 1] < off[i]) return false;
  return true;
}

template <int W>
static bool safe(const Words& x, std::random_device& rd) {
  uint32_t v[W];
  fill(v, W, half(x));
  return rsa::probably_prime<W>(v, 20, rd);
}

}  // namespace pbrsak
}  // namespace cb200

using namespace cb200;
using namespace cb200::pbrsak;

extern "C" {

int cb200_pbrsa_check_key(const uint8_t* N, size_t N_len, const uint8_t* p, size_t p_len, const uint8_t* q,
                          size_t q_len) {
  const char* fn = "cb200_pbrsa_check_key";
  Key k;
  int rc = parse_key(fn, N, N_len, p, p_len, q, q_len, nullptr, 0, false, &k);
  if (rc) return rc;
  std::random_device rd;
  for (const Words* x : {&k.p, &k.q}) {
    const int w = word_class(bitlen(*x), 32);
    const bool ok = w == 32 ? safe<32>(*x, rd) : w == 48 ? safe<48>(*x, rd) : safe<64>(*x, rd);
    if (!ok) {
      set_error("%s: %s is not a safe prime: (%s - 1) / 2 is composite", fn, x == &k.p ? "p" : "q",
                x == &k.p ? "p" : "q");
      return CB200_ERR_ARG;
    }
  }
  return 0;
}

int cb200_pbrsa_blind_sign(const uint8_t* N, size_t N_len, const uint8_t* p, size_t p_len, const uint8_t* q,
                           size_t q_len, const uint8_t* qinv, size_t qinv_len, const uint8_t* blinded,
                           const uint8_t* meta, const uint64_t* meta_off, uint8_t* sig, uint8_t* status, size_t n) {
  const char* fn = "cb200_pbrsa_blind_sign";
  Key k;
  int rc = parse_key(fn, N, N_len, p, p_len, q, q_len, qinv, qinv_len, true, &k);
  if (rc) return rc;
  if (!blinded || !meta || !meta_off || !sig || !status) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  if (!is_device_ptr(meta_off) && n) {
    if (!host_offsets_ok(meta_off, n)) {
      set_error("%s: meta_off decreases", fn);
      return CB200_ERR_ARG;
    }
    for (size_t i = 0; i < n; i++)
      if (bad_lengths(meta_off[i + 1] - meta_off[i], 0)) {
        set_error("%s: metadata %zu is longer than 2^31 - 8 bytes", fn, i);
        return CB200_ERR_ARG;
      }
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  return with_words(k.wp, k.m.wn,
                    [&](auto wp, auto wn) { return sign<wp, wn>(fn, k, blinded, meta, meta_off, sig, status, n); });
}

int cb200_pbrsa_verify(const uint8_t* N, size_t N_len, const uint8_t* msgs, const uint64_t* msg_off,
                       const uint8_t* meta, const uint64_t* meta_off, const uint8_t* sigs, uint8_t* status, size_t n) {
  const char* fn = "cb200_pbrsa_verify";
  if (!N) {
    set_error("%s: null key field", fn);
    return CB200_ERR_ARG;
  }
  Modulus m;
  int rc = parse_modulus(fn, N, N_len, &m);
  if (rc) return rc;
  if (!msgs || !msg_off || !meta || !meta_off || !sigs || !status) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  const bool dev = is_device_ptr(msgs);
  if (is_device_ptr(msg_off) != dev || is_device_ptr(meta) != dev || is_device_ptr(meta_off) != dev) {
    set_error("%s: mixed host/device pointers", fn);
    return CB200_ERR_ARG;
  }
  std::vector<uint8_t> framed;
  std::vector<uint64_t> off, mlen;
  if (!dev && n) {  // stage meta || msg per op as one string, with the metadata lengths as a row
    if (!host_offsets_ok(msg_off, n) || !host_offsets_ok(meta_off, n)) {
      set_error("%s: msg_off or meta_off decreases", fn);
      return CB200_ERR_ARG;
    }
    for (size_t i = 0; i < n; i++)
      if (bad_lengths(meta_off[i + 1] - meta_off[i], msg_off[i + 1] - msg_off[i])) {
        set_error("%s: op %zu: metadata and message together are longer than 2^31 - 8 bytes", fn, i);
        return CB200_ERR_ARG;
      }
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!dev) {
    framed.reserve((size_t)(msg_off[n] - msg_off[0] + meta_off[n] - meta_off[0]) + 1);
    off.resize(n + 1);
    mlen.resize(n);
    off[0] = 0;
    for (size_t i = 0; i < n; i++) {
      framed.insert(framed.end(), meta + meta_off[i], meta + meta_off[i + 1]);
      framed.insert(framed.end(), msgs + msg_off[i], msgs + msg_off[i + 1]);
      mlen[i] = meta_off[i + 1] - meta_off[i];
      off[i + 1] = framed.size();
    }
    framed.push_back(0);  // never empty
    msgs = framed.data();
    msg_off = off.data();
    meta = nullptr;
    meta_off = nullptr;
  }
  const uint64_t* ml = mlen.empty() ? nullptr : mlen.data();
  return with_words(m.wn, [&](auto wn) { return verify<wn>(fn, m, msgs, msg_off, meta, meta_off, ml, sigs, status, n); });
}

}  // extern "C"
