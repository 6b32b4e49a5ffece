// Threshold RSA signatures (the reference's tss/rsa package, Shoup's protocol 1): a signing party's shares of a batch of
// messages under its one key share, and the combination of k shares per op into the RSA signature, batched on the
// device with one thread per operation.  The arithmetic is rsa.cuh:
//   SignShare   tssrsa_sign_kernel<WN>      x^E mod N for the secret E = 2 Delta s_i, fixed 4-bit windows at WN words
//   Combine     tssrsa_combine_kernel<WN>   lambdas, prod xi^(2 lambda), one inverse, w^a x^b, y^e mod N == x
// WN is 64, 96 or 128 by N.  The key struct (N's Montgomery constants, E or e, Delta and (a, b)) is computed on the
// host once per call and copied into the call's level-1 work area.  Timed under the profiling class rsa.
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "rsa.cuh"
#include "rsa_host.h"

namespace cb200 {
namespace tssrsak {

template <int WN>
__global__ void __launch_bounds__(128) tssrsa_sign_kernel(const rsa::TssSignKey<WN>* __restrict__ K,
                                                          const uint8_t* __restrict__ in, size_t in_stride,
                                                          uint8_t* __restrict__ out, size_t out_stride, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rsa::tss_sign_share<WN>(out + i * out_stride, in + i * in_stride, *K);
}

// op i: k indices (uint16, host byte order) at idx + i idx_stride, k shares of kLen bytes at xi + i xi_stride, x at
// msg + i msg_stride
template <int WN>
__global__ void __launch_bounds__(128) tssrsa_combine_kernel(const rsa::TssCombineKey<WN>* __restrict__ K,
                                                             const uint8_t* __restrict__ idx, size_t idx_stride,
                                                             const uint8_t* __restrict__ xi, size_t xi_stride,
                                                             const uint8_t* __restrict__ msg, size_t msg_stride,
                                                             uint8_t* __restrict__ out, size_t out_stride,
                                                             uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint16_t* ix = (const uint16_t*)(idx + i * idx_stride);
  const uint8_t* x = xi + i * xi_stride;
  const int klen = K->klen;
  status[i] = (uint8_t)rsa::tss_combine<WN>(
      out + i * out_stride, [&](int t) -> uint32_t { return ix[t]; },
      [&](int t) { return x + (size_t)t * klen; }, msg + i * msg_stride, *K);
}

// ---------------------------------------------------------------- host side
using namespace rsah;

// Delta = players! as words
static Words factorial(int players) {
  Words d{1};
  for (int i = 2; i <= players; i++) d = mul(d, Words{(uint32_t)i});
  return d;
}
// players in 2 .. kTssMaxPlayers
static int check_players(const char* fn, int players) {
  if (players < 2 || players > rsa::kTssMaxPlayers) {
    set_error("%s: players is %d; 2 to %d are served", fn, players, rsa::kTssMaxPlayers);
    return CB200_ERR_ARG;
  }
  return 0;
}

template <int WN>
static int sign(const char* fn, const Modulus& m, const Words& E, int ebits, const uint8_t* digests, uint8_t* xi,
                size_t n) {
  rsa::TssSignKey<WN> K;
  load_mod<WN>(K.n, m.n);
  fill(K.e, WN + rsa::kDeltaWords, E);
  K.ebits = ebits;
  K.klen = m.klen;
  const size_t kl = (size_t)K.klen;
  Batch b{fn, n, xi, 1u << 14, 1u << 10, {{digests, kl, kl, kIn}, {xi, kl, kl, kOut}}, {}};
  return run_keyed(b, K, [&](const rsa::TssSignKey<WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    tssrsa_sign_kernel<WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r[0].p, r[0].stride, r[1].p, r[1].stride, cnt);
  });
}

// Host batches are staged by bytes: a row is k kLen + 2 k + kLen bytes in and kLen + 1 out, up to 33 KB at k = 64 and
// 4096 bits, so a chunk holds kChunkBytes of rows (at most 2^14 ops)
constexpr size_t kChunkBytes = (size_t)64 << 20;

template <int WN>
static int combine(const char* fn, const Modulus& m, uint32_t e, int players, int k, const uint8_t* idx,
                   const uint8_t* xi, const uint8_t* msgs, uint8_t* sig, uint8_t* status, size_t n) {
  rsa::TssCombineKey<WN> K;
  load_mod<WN>(K.n, m.n);
  K.e = e;
  const Words delta = factorial(players);
  fill(K.delta, rsa::kDeltaWords, delta);
  uint32_t ep[rsa::kEpWords];
  fill(ep, rsa::kEpWords, mul(mul(delta, delta), Words{4}));
  rsa::tss_bezout(&K.a, &K.a_neg, K.b, &K.b_neg, ep, e);
  K.a_bits = rsa::bits_of(&K.a, 1);
  K.b_bits = rsa::bits_of(K.b, rsa::kEpWords);
  K.k = k;
  K.klen = m.klen;
  const size_t kl = (size_t)K.klen, ki = 2 * (size_t)k, kx = (size_t)k * kl;
  const size_t chunk = std::max<size_t>(1, std::min<size_t>(1u << 14, kChunkBytes / (ki + kx + 2 * kl + 1)));
  Batch b{fn, n, sig, chunk, std::min<size_t>(chunk, 1u << 10),
          {{idx, ki, ki, kIn}, {xi, kx, kx, kIn}, {msgs, kl, kl, kIn}, {sig, kl, kl, kOut}, {status, 1, 1, kStatus}},
          {{!aligned({idx}, {}, 2), "%s: device idx must be 2-byte aligned"}}};
  return run_keyed(b, K, [&](const rsa::TssCombineKey<WN>* dk, const Rows& r, size_t cnt, cudaStream_t st) {
    tssrsa_combine_kernel<WN><<<blocks(cnt, 128), 128, 0, st>>>(dk, r[0].p, r[0].stride, r[1].p, r[1].stride, r[2].p,
                                                                r[2].stride, r[3].p, r[3].stride, r[4].p, cnt);
  });
}

}  // namespace tssrsak
}  // namespace cb200

using namespace cb200;
using namespace cb200::tssrsak;

extern "C" {

int cb200_tssrsa_sign_share(const uint8_t* N, size_t N_len, int players, const uint8_t* E, size_t E_len,
                            const uint8_t* digests, uint8_t* xi, size_t n) {
  const char* fn = "cb200_tssrsa_sign_share";
  if (!N || !E || !digests || !xi) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  Modulus m;
  int rc = parse_modulus(fn, N, N_len, &m);
  if (rc) return rc;
  rc = check_players(fn, players);
  if (rc) return rc;
  // E = 2 Delta s_i with s_i < (p - 1)(q - 1) / 4 < N / 4
  const Words E_w = be_words(E, E_len);
  const int ebits = m.nbits - 2 + bitlen(mul(factorial(players), Words{2}));
  if (bitlen(E_w) > ebits) {
    set_error("%s: the exponent has %d bits; 2 Delta s_i has at most %d", fn, bitlen(E_w), ebits);
    return CB200_ERR_ARG;
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  return with_words(m.wn, [&](auto wn) { return sign<wn>(fn, m, E_w, ebits, digests, xi, n); });
}

int cb200_tssrsa_combine(const uint8_t* N, size_t N_len, const uint8_t* e, size_t e_len, int players, int threshold,
                         int k, const uint16_t* idx, const uint8_t* xi, const uint8_t* msgs, uint8_t* sig,
                         uint8_t* status, size_t n) {
  const char* fn = "cb200_tssrsa_combine";
  if (!N || !e || !idx || !xi || !msgs || !sig || !status) {
    set_error("%s: null pointer", fn);
    return CB200_ERR_ARG;
  }
  Modulus m;
  int rc = parse_modulus(fn, N, N_len, &m);
  if (rc) return rc;
  const Words ew = be_words(e, e_len);
  if (ew.size() != 1 || ew[0] < 3 || !(ew[0] & 1)) {
    set_error("%s: the public exponent must be odd, at least 3 and below 2^32", fn);
    return CB200_ERR_ARG;
  }
  rc = check_players(fn, players);
  if (rc) return rc;
  if (threshold < 1 || threshold > players) {
    set_error("%s: threshold is %d; 1 to players (%d) are valid", fn, threshold, players);
    return CB200_ERR_ARG;
  }
  if (k < threshold || k > rsa::kTssMaxPlayers) {
    set_error("%s: k is %d shares; threshold (%d) to %d are served", fn, k, threshold, rsa::kTssMaxPlayers);
    return CB200_ERR_ARG;
  }
  rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  return with_words(m.wn, [&](auto wn) {
    return combine<wn>(fn, m, ew[0], players, k, (const uint8_t*)idx, xi, msgs, sig, status, n);
  });
}

}  // extern "C"
