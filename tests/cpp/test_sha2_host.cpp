// circl_b200/csrc/sha2.cuh compiled for the host: a line-oriented driver for tests/test_sha2_host.py.
// Each input line is "<op> <hex> ..." ("-" for an empty string) and produces one output line of hex:
//   sha256 <msg>                       SHA-256(msg)
//   hmac256 <key> <msg>                HMAC-SHA256(key, msg), key 32 bytes or "-" (the all-zero salt's constant pads)
//   hmac512 <key> <msg>                HMAC-SHA512(key, msg), key 64 bytes or "-"
//   extract <kem_id> <label> <ikm>     LabeledExtract("", label, ikm) of DHKEM kem_id (0x20: SHA-256, 0x21: SHA-512)
//   expand <kem_id> <prk> <label> <a> <b> <c> <L>
//                                      LabeledExpand(prk, label, a || b || c, L), the info read as three rows
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/sha2.cuh"

using namespace cb200;

static std::vector<uint8_t> unhex(std::string s) {
  if (s == "-") s.clear();
  std::vector<uint8_t> out(s.size() / 2 + 1, 0);
  for (size_t i = 0; i + 1 < s.size(); i += 2) out[i / 2] = (uint8_t)std::stoul(s.substr(i, 2), nullptr, 16);
  return out;
}
static int hlen(const std::string& s) { return s == "-" ? 0 : (int)(s.size() / 2); }

struct Bytes {  // a message from memory
  const uint8_t* p;
  uint8_t operator()(int j) const { return p[j]; }
};

template <class S>
static std::string hexd(const typename S::W (&h)[8], int n) {
  std::string out;
  char buf[3];
  for (int j = 0; j < n; j++) {
    snprintf(buf, sizeof buf, "%02x", sha2::digest_byte<S>(h, j));
    out += buf;
  }
  return out;
}
template <class S>
static void key_words(typename S::W (&k)[8], const std::vector<uint8_t>& b) {
  for (int i = 0; i < 8; i++) {
    k[i] = 0;
    for (int j = 0; j < S::kWordBytes; j++) k[i] = (k[i] << 8) | b[i * S::kWordBytes + j];
  }
}
template <class S>
static std::string hmac(const std::string& key, const std::string& msg) {
  typename S::W ki[8], ko[8], out[8];
  if (key == "-") {
    S::ipad0(ki);
    S::opad0(ko);
  } else {
    typename S::W k[8];
    key_words<S>(k, unhex(key));
    sha2::hmac_key<S>(ki, ko, k);
  }
  std::vector<uint8_t> m = unhex(msg);
  sha2::hmac<S>(out, ki, ko, hlen(msg), Bytes{m.data()});
  return hexd<S>(out, S::kDigest);
}
template <class S>
static std::string extract(int id, const std::string& label, const std::string& ikm) {
  std::vector<uint8_t> lab = unhex(label), in = unhex(ikm);
  std::string l(lab.begin(), lab.begin() + hlen(label));
  typename S::W prk[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, id, l.c_str(), hlen(label), in.data(), nullptr, nullptr, hlen(ikm), 0, 0});
  return hexd<S>(prk, S::kDigest);
}
template <class S>
static std::string expand(int id, const std::string& prkh, const std::string& label, const std::string& a,
                          const std::string& b, const std::string& c, int L) {
  std::vector<uint8_t> lab = unhex(label), va = unhex(a), vb = unhex(b), vc = unhex(c);
  std::string l(lab.begin(), lab.begin() + hlen(label));
  typename S::W prk[8], out[8];
  key_words<S>(prk, unhex(prkh));
  sha2::labeled_expand<S>(out, prk, sha2::Labeled{1, L, id, l.c_str(), hlen(label), va.data(), vb.data(), vc.data(),
                                                  hlen(a), hlen(b), hlen(c)});
  return hexd<S>(out, L);
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    std::string op;
    is >> op;
    if (op == "sha256") {
      std::string m;
      is >> m;
      std::vector<uint8_t> b = unhex(m);
      uint32_t h[8];
      sha2::Sha256::iv(h);
      sha2::absorb<sha2::Sha256>(h, 0, hlen(m), Bytes{b.data()});
      std::cout << hexd<sha2::Sha256>(h, 32) << "\n";
    } else if (op == "hmac256" || op == "hmac512") {
      std::string k, m;
      is >> k >> m;
      std::cout << (op == "hmac256" ? hmac<sha2::Sha256>(k, m) : hmac<sha2::Sha512>(k, m)) << "\n";
    } else if (op == "extract") {
      int id;
      std::string label, ikm;
      is >> std::hex >> id >> label >> ikm;
      std::cout << (id == 0x20 ? extract<sha2::Sha256>(id, label, ikm) : extract<sha2::Sha512>(id, label, ikm)) << "\n";
    } else if (op == "expand") {
      int id, L;
      std::string prk, label, a, b, c;
      is >> std::hex >> id >> prk >> label >> a >> b >> c >> std::dec >> L;
      std::cout << (id == 0x20 ? expand<sha2::Sha256>(id, prk, label, a, b, c, L)
                               : expand<sha2::Sha512>(id, prk, label, a, b, c, L))
                << "\n";
    } else {
      std::cout << "?\n";
    }
  }
  return 0;
}
