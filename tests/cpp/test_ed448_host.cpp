// circl_b200/csrc/ed448.cuh compiled for the host: a line-oriented driver for tests/test_ed448_host.py.
// Each input line is "<op> <hex> ..." ("-" for an empty string) and produces one output line of hex (or 0/1):
//   shake <ctx> <pre> <msg>        SHAKE256(dom4(ctx) || pre || msg, 114) through the three segments of the signing
//                                  hashes; ctx "none" for no dom4 string (the key-generation hash)
//   reduce <x, up to 120 bytes LE> x mod l
//   muladd <k> <s> <r>             (k s + r) mod l
//   canon <S, 57 bytes>            isLessThanOrder(S)
//   decode <A, 57 bytes>           1 + encode(decode(A)) if A decodes, else 0
//   keygen <seed>                  A
//   sign <seed> <A> <ctx> <msg>    R || S with A as given
//   verify <A> <ctx> <msg> <sig>   0 / 1
//   base <k, 56 bytes>             encode([k] G) for k < 2^447
//   basered <k, 56 bytes>          encode([k mod l] G) for any k < 2^448
//   dmul <s> <k> <A>               encode([s] G + [k] A), s < l, k < 2^448
//   madd|add|dbl <limbs>           one group-law formula on raw limbs (int32 LE words: P = X Y Z T, then the other
//                                  operand: x y dxy for madd, X Y Z dT for add), canonical X3 Y3 Z3 T3
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/ed448.cuh"

using namespace cb200;
using ed448::kW;

static std::vector<uint8_t> unhex(std::string s) {
  if (s == "-") s.clear();
  std::vector<uint8_t> out(s.size() / 2 + 8, 0);  // 8 bytes of read padding behind every message
  for (size_t i = 0; i + 1 < s.size(); i += 2) out[i / 2] = (uint8_t)std::stoul(s.substr(i, 2), nullptr, 16);
  return out;
}
static size_t hlen(const std::string& s) { return s == "-" ? 0 : s.size() / 2; }
template <int N>
static void words(uint32_t (&w)[N], const std::string& s) {
  std::vector<uint8_t> b = unhex(s);
  b.resize(4 * N + 8, 0);
  memcpy(w, b.data(), 4 * N);
}
static std::string hexb(const uint8_t* b, size_t n) {
  std::string out;
  char buf[3];
  for (size_t i = 0; i < n; i++) {
    snprintf(buf, sizeof buf, "%02x", b[i]);
    out += buf;
  }
  return out;
}
template <int N>
static std::string hex(const uint32_t (&w)[N]) {
  return hexb(reinterpret_cast<const uint8_t*>(w), 4 * N);
}
static std::string enc57(const ed448::GeExt& P) {
  uint32_t e[kW], top;
  ed448::ge_encode(e, top, P);
  uint8_t b[57];
  ed448::to_bytes57(b, e, top);
  return hexb(b, 57);
}
static void fe_from_limbs(x448::Fe& f, const uint8_t* p) { memcpy(f.v, p, 64); }
static std::string canon(const x448::Fe& f) {
  uint32_t w[kW];
  x448::fe_tobytes(w, f);
  return hex(w);
}

int main() {
  std::vector<int32_t> table(ed448::kTableWords);
  ed448::build_base_table(table.data());
  const int32_t* T = table.data();
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b, c, d;
    in >> op >> a >> b >> c >> d;
    if (op == "shake") {
      const bool none = a == "none";
      std::vector<uint8_t> ctx = unhex(none ? "-" : a), pre = unhex(b), m = unhex(c);
      uint64_t st[25];
      uint32_t h[30];
      ed448::shake256(st, ctx.data(), none ? -1 : (int32_t)hlen(a), pre.data(), (uint32_t)hlen(b), m.data(), hlen(c));
      ed448::lanes_to_words(h, st);
      printf("%s\n", hexb(reinterpret_cast<const uint8_t*>(h), 114).c_str());
    } else if (op == "reduce") {
      uint32_t x[30], r[kW];
      words(x, a);
      ed448::sc_reduce<30>(r, x);
      printf("%s\n", hex(r).c_str());
    } else if (op == "muladd") {
      uint32_t k[kW], s[kW], r[kW], S[kW];
      words(k, a);
      words(s, b);
      words(r, c);
      ed448::sc_muladd(S, k, s, r);
      printf("%s\n", hex(S).c_str());
    } else if (op == "canon") {
      uint32_t s[kW];
      words(s, a);
      printf("%d\n", ed448::sc_is_canonical(s, unhex(a)[56]) ? 1 : 0);
    } else if (op == "decode") {
      uint32_t A[kW];
      words(A, a);
      ed448::GeExt P;
      if (!ed448::ge_decode(P, A, unhex(a)[56])) {
        printf("0\n");
        continue;
      }
      printf("1%s\n", enc57(P).c_str());
    } else if (op == "keygen") {
      std::vector<uint8_t> seed = unhex(a);
      uint32_t A[kW], top;
      ed448::public_from_seed(A, top, seed.data(), T);
      uint8_t bb[57];
      ed448::to_bytes57(bb, A, top);
      printf("%s\n", hexb(bb, 57).c_str());
    } else if (op == "sign") {
      std::vector<uint8_t> seed = unhex(a), A = unhex(b), ctx = unhex(c), m = unhex(d);
      uint8_t sig[114];
      ed448::sign(sig, seed.data(), A.data(), ctx.data(), (int32_t)hlen(c), m.data(), hlen(d), T);
      printf("%s\n", hexb(sig, 114).c_str());
    } else if (op == "verify") {
      std::vector<uint8_t> A = unhex(a), ctx = unhex(b), m = unhex(c), sig = unhex(d);
      printf("%d\n", ed448::verify(A.data(), ctx.data(), (int32_t)hlen(b), m.data(), hlen(c), sig.data(), T) ? 1 : 0);
    } else if (op == "base" || op == "basered") {
      uint32_t k[kW];
      words(k, a);
      if (op == "basered") ed448::sc_reduce<kW>(k, k);
      ed448::GeExt P;
      ed448::ge_scalarmult_base(P, k, T);
      printf("%s\n", enc57(P).c_str());
    } else if (op == "dmul") {
      uint32_t s[kW], k[kW], A[kW];
      words(s, a);
      words(k, b);
      words(A, c);
      ed448::GeExt P, Q;
      if (!ed448::ge_decode(P, A, unhex(c)[56])) {
        printf("0\n");
        continue;
      }
      ed448::ge_double_mult(Q, s, k, P, T);
      printf("%s\n", enc57(Q).c_str());
    } else if (op == "madd" || op == "add" || op == "dbl") {
      std::vector<uint8_t> l = unhex(a);
      ed448::GeExt P, R;
      fe_from_limbs(P.X, &l[0]);
      fe_from_limbs(P.Y, &l[64]);
      fe_from_limbs(P.Z, &l[128]);
      fe_from_limbs(P.T, &l[192]);
      if (op == "madd") {
        ed448::GePre q;
        fe_from_limbs(q.x, &l[256]);
        fe_from_limbs(q.y, &l[320]);
        fe_from_limbs(q.dxy, &l[384]);
        ed448::ge_madd(R, P, q);
      } else if (op == "add") {
        ed448::GeCached q;
        fe_from_limbs(q.X, &l[256]);
        fe_from_limbs(q.Y, &l[320]);
        fe_from_limbs(q.Z, &l[384]);
        fe_from_limbs(q.dT, &l[448]);
        ed448::ge_add(R, P, q);
      } else {
        ed448::ge_dbl(R, P);
      }
      printf("%s %s %s %s\n", canon(R.X).c_str(), canon(R.Y).c_str(), canon(R.Z).c_str(), canon(R.T).c_str());
    } else {
      printf("?\n");
    }
  }
  return 0;
}
