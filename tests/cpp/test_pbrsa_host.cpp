// The partially blind RSA code of circl_b200/csrc/rsa.cuh compiled for the host, driven by tests/test_pbrsa_host.py:
// one command per stdin line, one result line each.  Numbers are big-endian hex of any length ("-" is the empty
// string); W, WP, WN are word counts.
//   derive WN N meta                      -> e' (derive_exponent, 2 WN bytes)
//   expw W m x e bits                     -> x^e mod m through exp_public_words (e < 2^bits, bits decimal)
//   half WP p e c                         -> c^d mod p through pb_half, d = e^-1 mod (p - 1) (p = 3 mod 4, e odd)
//   sign WP WN N p q qinv meta c          -> status s (pb_blind_sign; s is kLen bytes)
//   verify WN N meta msg sig              -> status (pb_verify)
//   prime W n                             -> 1 or 0 (probably_prime, 20 rounds)
#include <iostream>
#include <random>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/rsa.cuh"

using namespace cb200;
using Bytes = std::vector<uint8_t>;

static Bytes unhex(const std::string& s) {
  Bytes b;
  if (s == "-") return b;
  for (size_t i = 0; i + 1 < s.size(); i += 2) b.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return b;
}
static std::string hex(const uint8_t* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) s += d[p[i] >> 4], s += d[p[i] & 15];
  return n ? s : "-";
}
template <int W>
static void words(uint32_t* x, const std::string& h) {
  const Bytes b = unhex(h);
  rsa::from_be<W>(x, b.data(), (int)b.size());
}
template <int W>
static std::string whex(const uint32_t* x) {
  uint8_t b[4 * W];
  for (int i = 0; i < 4 * W; i++) b[i] = rsa::be_byte(x, 4 * W, i);
  return hex(b, 4 * W);
}
template <int W>
static rsa::Mod<W> mod(const std::string& h) {
  uint32_t m[W];
  words<W>(m, h);
  rsa::Mod<W> M;
  rsa::mod_init<W>(M, m);
  return M;
}
// (x - 1) / 2 of an odd x, and that minus 2
template <int W>
static void half_of(uint32_t* h, uint32_t* h2, const uint32_t* x) {
  for (int j = 0; j < W; j++) h[j] = (x[j] >> 1) | (j + 1 < W ? x[j + 1] << 31 : 0);
  uint32_t br = 2;
  for (int j = 0; j < W; j++) {
    h2[j] = h[j] - br;
    br = h[j] < br;
  }
}

// N as kLen bytes, its bit length, and the salt's pad states
struct NInfo {
  int nbits, klen;
  uint64_t si[8], so[8];
};
static NInfo ninfo(const std::string& h) {
  Bytes b = unhex(h);
  size_t i = 0;
  while (i < b.size() && !b[i]) i++;
  b.erase(b.begin(), b.begin() + i);
  NInfo r;
  int top = 8;
  while (!((b[0] >> (top - 1)) & 1)) top--;
  r.nbits = 8 * ((int)b.size() - 1) + top;
  r.klen = (int)b.size();
  rsa::pb_salt_states(r.si, r.so, b.data(), r.klen);
  return r;
}

template <int WN>
static std::string derive(std::istringstream& in) {
  std::string N, meta;
  in >> N >> meta;
  const NInfo ni = ninfo(N);
  const Bytes m = unhex(meta);
  uint32_t e[WN / 2];
  rsa::derive_exponent<WN>(e, ni.nbits, m.data(), (int)m.size(), ni.si, ni.so);
  return whex<WN / 2>(e);
}

template <int W>
static std::string expw(std::istringstream& in) {
  std::string mh, xh, eh;
  int bits;
  in >> mh >> xh >> eh >> bits;
  const rsa::Mod<W> M = mod<W>(mh);
  uint32_t x[W], e[W], r[W], one[W];
  words<W>(x, xh);
  words<W>(e, eh);
  for (int j = 0; j < W; j++) one[j] = j == 0;
  rsa::mont_mul<W>(x, x, M.r2, &M);
  rsa::exp_public_words<W>(r, x, e, bits, &M);
  rsa::mont_mul<W>(r, r, one, &M);
  return whex<W>(r);
}

template <int W>
static std::string half(std::istringstream& in) {
  std::string ph, eh, ch;
  in >> ph >> eh >> ch;
  const rsa::Mod<W> P = mod<W>(ph);
  uint32_t h[W], h2[W], e[W], c[W], r[W], one[W];
  half_of<W>(h, h2, P.m);
  rsa::Mod<W> H;
  rsa::mod_init<W>(H, h);
  words<W>(e, eh);
  words<W>(c, ch);
  for (int j = 0; j < W; j++) one[j] = j == 0;
  rsa::mont_mul<W>(c, c, P.r2, &P);
  rsa::pb_half<W>(r, c, e, P, H, h2);
  rsa::mont_mul<W>(r, r, one, &P);
  return whex<W>(r);
}

template <int WP, int WN>
static std::string sign(std::istringstream& in) {
  std::string N, p, q, qinv, meta, c;
  in >> N >> p >> q >> qinv >> meta >> c;
  static rsa::PbSignKey<WP, WN> K;
  K.p = mod<WP>(p);
  K.q = mod<WP>(q);
  uint32_t h[WP];
  half_of<WP>(h, K.ph2, K.p.m);
  rsa::mod_init<WP>(K.ph, h);
  half_of<WP>(h, K.qh2, K.q.m);
  rsa::mod_init<WP>(K.qh, h);
  words<WP>(K.qinv, qinv);
  K.n = mod<WN>(N);
  const NInfo ni = ninfo(N);
  for (int i = 0; i < 8; i++) K.si[i] = ni.si[i], K.so[i] = ni.so[i];
  K.klen = ni.klen;
  const Bytes cb = unhex(c), m = unhex(meta);
  Bytes out(K.klen);
  const uint32_t st = rsa::pb_blind_sign<WP, WN>(out.data(), cb.data(), m.data(), (int)m.size(), K);
  return std::to_string(st) + " " + hex(out.data(), out.size());
}

template <int WN>
static std::string verify(std::istringstream& in) {
  std::string N, meta, msg, sig;
  in >> N >> meta >> msg >> sig;
  static rsa::PbVerifyKey<WN> K;
  K.n = mod<WN>(N);
  const NInfo ni = ninfo(N);
  for (int i = 0; i < 8; i++) K.si[i] = ni.si[i], K.so[i] = ni.so[i];
  K.klen = ni.klen;
  const Bytes md = unhex(meta), m = unhex(msg), s = unhex(sig);
  return std::to_string(rsa::pb_verify<WN>(m.data(), (int)m.size(), md.data(), (int)md.size(), s.data(), K));
}

template <int W>
static std::string prime(std::istringstream& in) {
  std::string nh;
  in >> nh;
  uint32_t n[W];
  words<W>(n, nh);
  static std::mt19937 rng(5);
  return rsa::probably_prime<W>(n, 20, rng) ? "1" : "0";
}

static std::string run(const std::string& line) {
  std::istringstream in(line);
  std::string op;
  int w, w2 = 0;
  in >> op >> w;
  if (op == "derive" || op == "verify") {
    switch (w) {
      case 64: return op == "derive" ? derive<64>(in) : verify<64>(in);
      case 96: return op == "derive" ? derive<96>(in) : verify<96>(in);
      case 128: return op == "derive" ? derive<128>(in) : verify<128>(in);
    }
  } else if (op == "expw") {
    switch (w) {
      case 32: return expw<32>(in);
      case 48: return expw<48>(in);
      case 64: return expw<64>(in);
      case 96: return expw<96>(in);
      case 128: return expw<128>(in);
    }
  } else if (op == "half" || op == "prime") {
    switch (w) {
      case 32: return op == "half" ? half<32>(in) : prime<32>(in);
      case 48: return op == "half" ? half<48>(in) : prime<48>(in);
      case 64: return op == "half" ? half<64>(in) : prime<64>(in);
    }
  } else if (op == "sign") {
    in >> w2;
    switch (w * 1000 + w2) {
      case 32064: return sign<32, 64>(in);
      case 48064: return sign<48, 64>(in);
      case 48096: return sign<48, 96>(in);
      case 64064: return sign<64, 64>(in);
      case 64096: return sign<64, 96>(in);
      case 64128: return sign<64, 128>(in);
    }
  }
  return "?";
}

int main() {
  std::string l;
  while (std::getline(std::cin, l)) std::cout << run(l) << "\n";
  return 0;
}
