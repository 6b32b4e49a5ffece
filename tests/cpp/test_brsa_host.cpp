// circl_b200/csrc/rsa.cuh compiled for the host, driven by tests/test_brsa_host.py: one command per stdin line, one
// result line each.  Numbers are big-endian hex of any length ("-" is the empty string); W, WP, WN are word counts.
//   mul W m a b                       -> a b R^-1 mod m (Montgomery product, R = 2^(32 W)), 4 W bytes
//   exps W m x d                      -> x^d mod m through exp_secret (d < m)
//   expp W m x e                      -> x^e mod m through exp_public (e a decimal below 2^32)
//   sign WP WN N e p q dp dq qinv c   -> status s (blind_sign; s is kLen bytes)
//   verify WN slen N e msg sig        -> status (verify)
#include <cstdio>
#include <iostream>
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

template <int W>
static std::string arith(const std::string& op, std::istringstream& in) {
  std::string mh, xh, yh;
  in >> mh >> xh >> yh;
  const rsa::Mod<W> M = mod<W>(mh);
  uint32_t x[W], y[W], r[W], one[W];
  words<W>(x, xh);
  for (int j = 0; j < W; j++) one[j] = j == 0;
  if (op == "mul") {
    words<W>(y, yh);
    rsa::mont_mul<W>(r, x, y, &M);
    return whex<W>(r);
  }
  rsa::mont_mul<W>(x, x, M.r2, &M);
  if (op == "exps") {
    words<W>(y, yh);
    rsa::exp_secret<W>(r, x, y, &M);
  } else {
    rsa::exp_public<W>(r, x, (uint32_t)std::stoul(yh), &M);
  }
  rsa::mont_mul<W>(r, r, one, &M);
  return whex<W>(r);
}

static uint32_t u32(const std::string& h) {
  const Bytes b = unhex(h);
  uint32_t v = 0;
  for (uint8_t c : b) v = v << 8 | c;
  return v;
}
static int nbytes(const std::string& h) {
  const Bytes b = unhex(h);
  size_t i = 0;
  while (i < b.size() && !b[i]) i++;
  int bits = 0;
  if (i < b.size())
    for (bits = 8; !((b[i] >> (bits - 1)) & 1); bits--) {
    }
  return (int)(b.size() - i - 1) * 8 + bits;
}

template <int WP, int WN>
static std::string sign(std::istringstream& in) {
  std::string N, e, p, q, dp, dq, qinv, c;
  in >> N >> e >> p >> q >> dp >> dq >> qinv >> c;
  static rsa::SignKey<WP, WN> K;
  K.p = mod<WP>(p);
  K.q = mod<WP>(q);
  words<WP>(K.dp, dp);
  words<WP>(K.dq, dq);
  words<WP>(K.qinv, qinv);
  K.n = mod<WN>(N);
  K.e = u32(e);
  K.klen = (nbytes(N) + 7) / 8;
  const Bytes cb = unhex(c);
  Bytes out(K.klen);
  const uint32_t st = rsa::blind_sign<WP, WN>(out.data(), cb.data(), K);
  return std::to_string(st) + " " + hex(out.data(), out.size());
}

template <int WN>
static std::string verify(std::istringstream& in) {
  std::string slen, N, e, msg, sig;
  in >> slen >> N >> e >> msg >> sig;
  static rsa::VerifyKey<WN> K;
  K.n = mod<WN>(N);
  K.e = u32(e);
  K.klen = (nbytes(N) + 7) / 8;
  K.slen = std::stoi(slen);
  const Bytes m = unhex(msg), s = unhex(sig);
  return std::to_string(rsa::verify<WN>(m.data(), m.size(), s.data(), K));
}

static std::string run(const std::string& line) {
  std::istringstream in(line);
  std::string op;
  int w, w2 = 0;
  in >> op >> w;
  if (op == "mul" || op == "exps" || op == "expp") {
    switch (w) {
      case 32: return arith<32>(op, in);
      case 48: return arith<48>(op, in);
      case 64: return arith<64>(op, in);
      case 96: return arith<96>(op, in);
      case 128: return arith<128>(op, in);
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
  } else if (op == "verify") {
    switch (w) {
      case 64: return verify<64>(in);
      case 96: return verify<96>(in);
      case 128: return verify<128>(in);
    }
  }
  return "?";
}

int main() {
  std::string l;
  while (std::getline(std::cin, l)) std::cout << run(l) << "\n";
  return 0;
}
