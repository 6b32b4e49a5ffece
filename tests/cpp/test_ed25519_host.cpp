// circl_b200/csrc/ed25519.cuh compiled for the host: a line-oriented driver for tests/test_ed25519_host.py.
// Each input line is "<op> <hex> ..." and produces one output line of hex (or 0/1):
//   sha512 <msg>                 SHA-512(msg), msg of at least 32 bytes: its first 32 or 64 bytes go through the
//                                prefix path of the signing hashes, the rest through the message path
//   reduce <x, 64 bytes LE>      x mod L
//   muladd <r> <k> <a>           (r + k a) mod L
//   canon <S>                    isLessThanOrder(S)
//   decode <A>                   1 + encode(decode(A)) if A decodes, else 0
//   keygen <seed>                A
//   sign <seed> <A> <msg>        R || S with A as given
//   verify <A> <msg> <R||S>      0 / 1
//   base <k>                     encode([k] B) for k < 2^255
//   dmul <s> <k> <A>             encode([s] B + [k] A)
//   x25519 <k>                   X25519 KeyGen through the fixed-base core, then through the ladder on u = 9
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/ed25519.cuh"

using namespace cb200;

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> out(s.size() / 2 + 8, 0);  // 8 bytes of read padding behind every message
  for (size_t i = 0; i + 1 < s.size(); i += 2) out[i / 2] = (uint8_t)std::stoul(s.substr(i, 2), nullptr, 16);
  out.resize(s.size() / 2 + 8);
  return out;
}
template <int N>
static void words(uint32_t (&w)[N], const std::string& s) {
  std::vector<uint8_t> b = unhex(s);
  memcpy(w, b.data(), 4 * N);
}
template <int N>
static std::string hex(const uint32_t (&w)[N]) {
  std::string out;
  char buf[3];
  const uint8_t* b = reinterpret_cast<const uint8_t*>(w);
  for (int i = 0; i < 4 * N; i++) {
    snprintf(buf, sizeof buf, "%02x", b[i]);
    out += buf;
  }
  return out;
}

int main() {
  std::vector<int32_t> table(x25519::kBaseTableWords);
  x25519::build_base_table(table.data());
  const int32_t* T = table.data();
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b, c;
    in >> op >> a >> b >> c;
    if (op == "sha512") {
      if (a == "-") a.clear();
      std::vector<uint8_t> m = unhex(a);
      uint32_t out[16];
      if (a.size() / 2 >= 64) {
        uint32_t pre[16];
        memcpy(pre, m.data(), 64);
        ed25519::sha512<8>(out, pre, m.data() + 64, a.size() / 2 - 64);
      } else if (a.size() / 2 >= 32) {
        uint32_t pre[8];
        memcpy(pre, m.data(), 32);
        ed25519::sha512<4>(out, pre, m.data() + 32, a.size() / 2 - 32);
      } else {
        printf("skip\n");
        continue;
      }
      printf("%s\n", hex(out).c_str());
    } else if (op == "reduce") {
      uint32_t x[16], r[8];
      words(x, a);
      ed25519::sc_reduce(r, x);
      printf("%s\n", hex(r).c_str());
    } else if (op == "muladd") {
      uint32_t r[8], k[8], s[8], S[8];
      words(r, a);
      words(k, b);
      words(s, c);
      ed25519::sc_muladd(S, r, k, s);
      printf("%s\n", hex(S).c_str());
    } else if (op == "canon") {
      uint32_t s[8];
      words(s, a);
      printf("%d\n", ed25519::sc_is_canonical(s) ? 1 : 0);
    } else if (op == "decode") {
      uint32_t A[8], e[8];
      words(A, a);
      x25519::GeExt P;
      if (!ed25519::ge_decode(P, A)) {
        printf("0\n");
        continue;
      }
      ed25519::ge_encode(e, P);
      printf("1%s\n", hex(e).c_str());
    } else if (op == "keygen") {
      uint32_t seed[8], A[8];
      words(seed, a);
      ed25519::public_from_seed(A, seed, T);
      printf("%s\n", hex(A).c_str());
    } else if (op == "sign") {
      uint32_t seed[8], A[8], R[8], S[8];
      words(seed, a);
      words(A, b);
      if (c == "-") c.clear();
      std::vector<uint8_t> m = unhex(c);
      ed25519::sign(R, S, seed, A, m.data(), c.size() / 2, T);
      printf("%s%s\n", hex(R).c_str(), hex(S).c_str());
    } else if (op == "verify") {
      uint32_t A[8], R[8], S[8];
      words(A, a);
      if (b == "-") b.clear();
      std::vector<uint8_t> m = unhex(b), sig = unhex(c);
      memcpy(R, sig.data(), 32);
      memcpy(S, sig.data() + 32, 32);
      printf("%d\n", ed25519::verify(A, m.data(), b.size() / 2, R, S, T) ? 1 : 0);
    } else if (op == "base") {
      uint32_t k[8], e[8];
      words(k, a);
      x25519::GeExt P;
      x25519::ge_scalarmult_base(P, k, T);
      ed25519::ge_encode(e, P);
      printf("%s\n", hex(e).c_str());
    } else if (op == "dmul") {
      uint32_t s[8], k[8], A[8], e[8];
      words(s, a);
      words(k, b);
      words(A, c);
      x25519::GeExt P, Q;
      if (!ed25519::ge_decode(P, A)) {
        printf("0\n");
        continue;
      }
      ed25519::ge_double_mult(Q, s, k, P, T);
      ed25519::ge_encode(e, Q);
      printf("%s\n", hex(e).c_str());
    } else if (op == "x25519") {
      uint32_t k[8], u1[8], u2[8], nine[8] = {9, 0, 0, 0, 0, 0, 0, 0};
      words(k, a);
      x25519::scalarmult_base(u1, k, T);
      x25519::scalarmult(u2, k, nine);
      printf("%s %s\n", hex(u1).c_str(), hex(u2).c_str());
    } else {
      printf("?\n");
    }
  }
  return 0;
}
