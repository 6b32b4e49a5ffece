// circl_b200/csrc/sha2.cuh's SHA-384 and two-block HKDF-Expand compiled for the host: a line-oriented driver for
// tests/test_sha384_host.py.  Each input line produces one output line of hex ("-" for an empty string):
//   sha384 <msg>                        SHA-384(msg)
//   hmac384 <key> <msg>                 HMAC-SHA384(key, msg), key 48 bytes or "-" (the all-zero salt's constant pads)
//   extract <kem_id> <label> <ikm>      LabeledExtract("", label, ikm) (0x11: SHA-384, 0x12: SHA-512)
//   expand2 <kem_id> <prk> <label> <info> <L>
//                                       LabeledExpand(prk, label, info, L) for L up to two digests: T(1) || T(2),
//                                       T(2) from ExpandNext
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
static std::string hex_digest(const typename S::W (&h)[8], int n) {
  std::string s;
  char t[3];
  for (int j = 0; j < n; j++) snprintf(t, 3, "%02x", sha2::digest_byte<S>(h, j)), s += t;
  return s;
}
template <class S>
static void key_words(typename S::W (&k)[8], const std::vector<uint8_t>& b) {
  for (int i = 0; i < 8; i++) k[i] = 0;
  for (int j = 0; j < S::kDigest; j++) k[j / S::kWordBytes] |= (typename S::W)b[j] << (8 * (S::kWordBytes - 1 - j % S::kWordBytes));
}
static const char* literal(const std::string& s) {  // labels must outlive the Labeled that points at them
  static std::vector<std::string> keep;
  keep.push_back(s);
  return keep.back().c_str();
}
template <class S>
static std::string extract(int id, const std::string& label, const std::string& ikm) {
  const std::vector<uint8_t> m = unhex(ikm);
  typename S::W prk[8];
  sha2::labeled_extract<S>(prk, sha2::Labeled{0, 0, id, literal(label), (int)label.size(), m.data(), nullptr, nullptr,
                                              hlen(ikm), 0, 0});
  return hex_digest<S>(prk, S::kDigest);
}
template <class S>
static std::string expand2(int id, const std::string& prkh, const std::string& label, const std::string& info, int L) {
  const std::vector<uint8_t> p = unhex(prkh), inf = unhex(info);
  typename S::W prk[8], ki[8], ko[8], t1[8], t2[8];
  key_words<S>(prk, p);
  sha2::hmac_key<S>(ki, ko, prk);
  const sha2::Labeled m{1, L, id, literal(label), (int)label.size(), inf.data(), nullptr, nullptr, hlen(info), 0, 0};
  sha2::hmac<S>(t1, ki, ko, m.len(), m);
  const sha2::ExpandNext<S, sha2::Labeled> m2{t1, m};
  sha2::hmac<S>(t2, ki, ko, m2.len(), m2);
  return hex_digest<S>(t1, S::kDigest) + hex_digest<S>(t2, S::kDigest);
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    in >> op;
    if (op == "sha384") {
      std::string m;
      in >> m;
      const std::vector<uint8_t> b = unhex(m);
      uint64_t h[8];
      sha2::Sha384::iv(h);
      sha2::absorb<sha2::Sha384>(h, 0, hlen(m), Bytes{b.data()});
      std::cout << hex_digest<sha2::Sha384>(h, 48) << "\n";
    } else if (op == "hmac384") {
      std::string k, m;
      in >> k >> m;
      const std::vector<uint8_t> kb = unhex(k), mb = unhex(m);
      uint64_t ki[8], ko[8], key[8], out[8];
      if (k == "-") {
        sha2::Sha384::ipad0(ki);
        sha2::Sha384::opad0(ko);
      } else {
        key_words<sha2::Sha384>(key, kb);
        sha2::hmac_key<sha2::Sha384>(ki, ko, key);
      }
      sha2::hmac<sha2::Sha384>(out, ki, ko, hlen(m), Bytes{mb.data()});
      std::cout << hex_digest<sha2::Sha384>(out, 48) << "\n";
    } else if (op == "extract") {
      int id;
      std::string label, ikm;
      in >> std::hex >> id >> label >> ikm;
      std::cout << (id == 0x11 ? extract<sha2::Sha384>(id, label, ikm) : extract<sha2::Sha512>(id, label, ikm)) << "\n";
    } else if (op == "expand2") {
      int id, L;
      std::string prk, label, info;
      in >> std::hex >> id >> prk >> label >> info >> std::dec >> L;
      std::cout << (id == 0x11 ? expand2<sha2::Sha384>(id, prk, label, info, L)
                               : expand2<sha2::Sha512>(id, prk, label, info, L)) << "\n";
    } else {
      std::cerr << "unknown op " << op << "\n";
      return 1;
    }
  }
  return 0;
}
