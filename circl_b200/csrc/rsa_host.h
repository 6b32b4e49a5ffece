// Host side of the RSA entry points (brsa.cu, pbrsa.cu): multi-precision values as word vectors, the word counts that
// serve a key, the checks of the modulus and its two primes, the key structs' CRT part, and the launch of a batch
// under the call's key.
#pragma once
#include <algorithm>
#include <cstdint>
#include <type_traits>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "rsa.cuh"

namespace cb200 {
namespace rsah {

using Words = std::vector<uint32_t>;  // little-endian, without leading zero words

inline Words be_words(const uint8_t* s, size_t len) {
  Words w((len + 3) / 4, 0);
  for (size_t i = 0; i < len; i++) {
    const size_t k = len - 1 - i;
    w[k / 4] |= (uint32_t)s[i] << (8 * (k % 4));
  }
  while (!w.empty() && !w.back()) w.pop_back();
  return w;
}
inline int bitlen(const Words& w) {
  if (w.empty()) return 0;
  int b = 32;
  while (!((w.back() >> (b - 1)) & 1)) b--;
  return 32 * ((int)w.size() - 1) + b;
}
inline Words mul(const Words& a, const Words& b) {
  Words r(a.size() + b.size(), 0);
  for (size_t i = 0; i < a.size(); i++) {
    uint64_t c = 0;
    for (size_t j = 0; j < b.size(); j++) {
      c += (uint64_t)a[i] * b[j] + r[i + j];
      r[i + j] = (uint32_t)c;
      c >>= 32;
    }
    r[i + b.size()] = (uint32_t)c;
  }
  while (!r.empty() && !r.back()) r.pop_back();
  return r;
}
// a < b for values without leading zero words
inline bool less(const Words& a, const Words& b) {
  if (a.size() != b.size()) return a.size() < b.size();
  return std::lexicographical_compare(a.rbegin(), a.rend(), b.rbegin(), b.rend());
}
// the word count serving a modulus of `bits` bits: 32, 48, 64 (primes) or 64, 96, 128 (N); 0 past the largest
inline int word_class(int bits, int unit) {
  for (int w = unit; w <= 2 * unit; w += unit / 2)
    if (bits <= 32 * w) return w;
  return 0;
}
inline void fill(uint32_t* dst, int W, const Words& w) {
  for (int j = 0; j < W; j++) dst[j] = j < (int)w.size() ? w[j] : 0;
}

struct Modulus {
  Words n;
  int nbits, klen, wn;
};
// N (not null) of 2048 to 4096 bits
inline int parse_modulus(const char* fn, const uint8_t* N, size_t N_len, Modulus* m) {
  m->n = be_words(N, N_len);
  m->nbits = bitlen(m->n);
  if (m->nbits < 2048 || m->nbits > 4096) {
    set_error("%s: the modulus has %d bits; 2048 to 4096 are served", fn, m->nbits);
    return CB200_ERR_ARG;
  }
  m->klen = (m->nbits + 7) / 8;
  m->wn = word_class(m->nbits, 64);
  return 0;
}

// p and q (not null): two odd numbers above 2 with p q = N, the larger of at most 2048 bits; *wp its word count
inline int parse_primes(const char* fn, const Words& n, const uint8_t* P, size_t P_len, const uint8_t* Q, size_t Q_len,
                        Words* p, Words* q, int* wp) {
  *p = be_words(P, P_len);
  *q = be_words(Q, Q_len);
  if (p->empty() || q->empty() || !((*p)[0] & 1) || !((*q)[0] & 1) || mul(*p, *q) != n || bitlen(*p) < 2 ||
      bitlen(*q) < 2) {
    set_error("%s: the key is not two odd primes p, q with p q = N", fn);
    return CB200_ERR_ARG;
  }
  *wp = word_class(std::max(bitlen(*p), bitlen(*q)), 32);
  if (!*wp) {
    set_error("%s: the larger prime has %d bits; at most 2048 are served", fn, std::max(bitlen(*p), bitlen(*q)));
    return CB200_ERR_ARG;
  }
  return 0;
}

// a word count as a type, so that a generic lambda can use it as a template argument
template <int W>
using WordCount = std::integral_constant<int, W>;
// f(WP, WN) for the word counts of a sign key: the five served pairs below, else (64, 128)
template <class F>
int with_words(int wp, int wn, const F& f) {
  switch (wp * 1000 + wn) {
    case 32064: return f(WordCount<32>(), WordCount<64>());
    case 48064: return f(WordCount<48>(), WordCount<64>());
    case 48096: return f(WordCount<48>(), WordCount<96>());
    case 64064: return f(WordCount<64>(), WordCount<64>());
    case 64096: return f(WordCount<64>(), WordCount<96>());
    default: return f(WordCount<64>(), WordCount<128>());
  }
}
// f(WN) for the word count of N: 64, 96, else 128
template <class F>
int with_words(int wn, const F& f) {
  switch (wn) {
    case 64: return f(WordCount<64>());
    case 96: return f(WordCount<96>());
    default: return f(WordCount<128>());
  }
}

// M of the value x (at most W words)
template <int W>
void load_mod(rsa::Mod<W>& M, const Words& x) {
  uint32_t w[W];
  fill(w, W, x);
  rsa::mod_init<W>(M, w);
}
// the CRT part of a sign key (rsa::SignKey or rsa::PbSignKey): p, q, qinv, N and klen
template <int WP, int WN, class Key>
void load_crt(Key& K, const Modulus& m, const Words& p, const Words& q, const Words& qinv) {
  load_mod<WP>(K.p, p);
  load_mod<WP>(K.q, q);
  fill(K.qinv, WP, qinv);
  load_mod<WN>(K.n, m.n);
  K.klen = m.klen;
}

inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

// run_batch under the call's key K: every sub-batch copies K into its slot's level-1 work area and starts its kernel
// by launch(dk, rows, count, st) with dk the device copy, timed under the profiling class rsa
template <class Key, class Launch>
int run_keyed(const Batch& b, const Key& K, const Launch& launch) {
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    int rc = arena(slot, sizeof(Key), &A);
    if (rc) return rc;
    Key* dk = (Key*)A.take(sizeof(Key));
    CB200_CUDA(cudaMemcpyAsync(dk, &K, sizeof(Key), cudaMemcpyHostToDevice, st));
    {
      KernelScope ks(KID_RSA, st);
      launch(dk, r, cnt, st);
    }
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

}  // namespace rsah
}  // namespace cb200
