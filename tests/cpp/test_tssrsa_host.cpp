// The threshold RSA code of circl_b200/csrc/rsa.cuh compiled for the host, driven by tests/test_tssrsa_host.py: one
// command per stdin line, one result line each.  Numbers are big-endian hex of any length; W, WN are word counts.
//   inv W m x                        -> x^-1 mod m, or "none" (mod_inverse on x R mod m)
//   lambda l j1,j2,..                -> "1", or "0" and each lambda as a signed hex (tss_lambda, Delta = l!)
//   bezout l e                       -> a b as signed hex (tss_bezout of e' = 4 (l!)^2 and e)
//   sign WN N ebits E x              -> x^E mod N, kLen bytes (tss_sign_share)
//   combine WN N e l j1,j2,.. xi x   -> status y (tss_combine; xi is k rows of kLen bytes, x kLen bytes)
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/rsa.cuh"

using namespace cb200;
using Bytes = std::vector<uint8_t>;

static Bytes unhex(const std::string& s) {
  Bytes b;
  for (size_t i = 0; i + 1 < s.size(); i += 2) b.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return b;
}
static std::string hex(const uint8_t* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) s += d[p[i] >> 4], s += d[p[i] & 15];
  return s;
}
template <int W>
static void words(uint32_t* x, const std::string& h) {
  const Bytes b = unhex(h);
  rsa::from_be<W>(x, b.data(), (int)b.size());
}
static std::string whex(const uint32_t* x, int n) {
  std::vector<uint8_t> b(4 * n);
  for (int i = 0; i < 4 * n; i++) b[i] = rsa::be_byte(x, 4 * n, i);
  return hex(b.data(), b.size());
}
static std::vector<uint32_t> csv(const std::string& s) {
  std::vector<uint32_t> v;
  std::stringstream ss(s);
  std::string t;
  while (std::getline(ss, t, ',')) v.push_back((uint32_t)std::stoul(t));
  return v;
}
static void factorial(uint32_t* d, int l) {
  for (int j = 0; j < rsa::kDeltaWords; j++) d[j] = j == 0;
  for (int i = 2; i <= l; i++) {
    uint64_t c = 0;
    for (int j = 0; j < rsa::kDeltaWords; j++) {
      c += (uint64_t)d[j] * i;
      d[j] = (uint32_t)c;
      c >>= 32;
    }
  }
}

template <int W>
static std::string inv(std::istringstream& in) {
  std::string hm, hx;
  in >> hm >> hx;
  uint32_t m[W], x[W], r[W], one[W];
  words<W>(m, hm);
  words<W>(x, hx);
  rsa::Mod<W> M;
  rsa::mod_init<W>(M, m);
  for (int j = 0; j < W; j++) one[j] = j == 0;
  rsa::mont_mul<W>(x, x, M.r2, &M);
  if (!rsa::mod_inverse<W>(r, x, &M)) return "none";
  rsa::mont_mul<W>(r, r, one, &M);
  return whex(r, W);
}

template <int WN>
static std::string sign(std::istringstream& in) {
  std::string hn, he, hx;
  int ebits;
  in >> hn >> ebits >> he >> hx;
  static rsa::TssSignKey<WN> K;
  uint32_t n[WN];
  words<WN>(n, hn);
  rsa::mod_init<WN>(K.n, n);
  words<WN + rsa::kDeltaWords>(K.e, he);
  K.ebits = ebits;
  K.klen = (K.n.bits + 7) / 8;
  const Bytes x = unhex(hx);
  Bytes out(K.klen);
  rsa::tss_sign_share<WN>(out.data(), x.data(), K);
  return hex(out.data(), out.size());
}

template <int WN>
static std::string combine(std::istringstream& in) {
  std::string hn, he, hj, hxi, hx;
  int l;
  in >> hn >> he >> l >> hj >> hxi >> hx;
  static rsa::TssCombineKey<WN> K;
  uint32_t n[WN];
  words<WN>(n, hn);
  rsa::mod_init<WN>(K.n, n);
  K.e = (uint32_t)std::stoul(he, nullptr, 16);
  factorial(K.delta, l);
  uint32_t d2[2 * rsa::kDeltaWords] = {0}, ep[rsa::kEpWords];
  for (int i = 0; i < rsa::kDeltaWords; i++) {
    uint64_t c = 0;
    for (int j = 0; j < rsa::kDeltaWords; j++) {
      c += (uint64_t)K.delta[i] * K.delta[j] + d2[i + j];
      d2[i + j] = (uint32_t)c;
      c >>= 32;
    }
    d2[i + rsa::kDeltaWords] = (uint32_t)c;
  }
  for (int j = 0; j < rsa::kEpWords; j++) ep[j] = (d2[j] << 2) | (j ? d2[j - 1] >> 30 : 0);
  rsa::tss_bezout(&K.a, &K.a_neg, K.b, &K.b_neg, ep, K.e);
  K.a_bits = rsa::bits_of(&K.a, 1);
  K.b_bits = rsa::bits_of(K.b, rsa::kEpWords);
  const std::vector<uint32_t> idx = csv(hj);
  K.k = (int)idx.size();
  K.klen = (K.n.bits + 7) / 8;
  const Bytes xi = unhex(hxi), x = unhex(hx);
  Bytes out(K.klen);
  const uint32_t st = rsa::tss_combine<WN>(
      out.data(), [&](int t) { return idx[t]; }, [&](int t) { return xi.data() + (size_t)t * K.klen; }, x.data(), K);
  return std::to_string(st) + " " + hex(out.data(), out.size());
}

template <class F>
static std::string by_words(int w, const F& f) {
  switch (w) {
    case 64: return f(std::integral_constant<int, 64>());
    case 96: return f(std::integral_constant<int, 96>());
    default: return f(std::integral_constant<int, 128>());
  }
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    int w = 0;
    in >> cmd;
    if (cmd == "inv") {
      in >> w;
      std::cout << by_words(w, [&](auto W) { return inv<W>(in); }) << "\n";
    } else if (cmd == "lambda") {
      int l;
      std::string hj;
      in >> l >> hj;
      const std::vector<uint32_t> idx = csv(hj);
      uint32_t delta[rsa::kDeltaWords], lam[rsa::kLambdaWords];
      factorial(delta, l);
      std::string res = "0";
      for (int t = 0; t < (int)idx.size(); t++) {
        bool neg = false;
        if (rsa::tss_lambda(lam, &neg, [&](int u) { return idx[u]; }, t, (int)idx.size(), delta)) {
          res = "1";
          break;
        }
        res += std::string(" ") + (neg ? "-" : "+") + whex(lam, rsa::kLambdaWords);
      }
      std::cout << res << "\n";
    } else if (cmd == "bezout") {
      int l;
      uint32_t e;
      in >> l >> e;
      uint32_t d[rsa::kDeltaWords], ep[rsa::kEpWords] = {0}, a, b[rsa::kEpWords];
      int an, bn;
      factorial(d, l);
      // e' = 4 d^2 (d < 2^297)
      uint32_t d2[2 * rsa::kDeltaWords] = {0};
      for (int i = 0; i < rsa::kDeltaWords; i++) {
        uint64_t c = 0;
        for (int j = 0; j < rsa::kDeltaWords; j++) {
          c += (uint64_t)d[i] * d[j] + d2[i + j];
          d2[i + j] = (uint32_t)c;
          c >>= 32;
        }
        d2[i + rsa::kDeltaWords] = (uint32_t)c;
      }
      for (int j = 0; j < rsa::kEpWords; j++) ep[j] = (d2[j] << 2) | (j ? d2[j - 1] >> 30 : 0);
      rsa::tss_bezout(&a, &an, b, &bn, ep, e);
      std::cout << (an ? "-" : "+") << whex(&a, 1) << " " << (bn ? "-" : "+") << whex(b, rsa::kEpWords) << "\n";
    } else if (cmd == "sign") {
      in >> w;
      std::cout << by_words(w, [&](auto W) { return sign<W>(in); }) << "\n";
    } else if (cmd == "combine") {
      in >> w;
      std::cout << by_words(w, [&](auto W) { return combine<W>(in); }) << "\n";
    } else {
      std::cout << "?\n";
    }
  }
  return 0;
}
