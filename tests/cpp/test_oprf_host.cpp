// circl_b200/csrc/oprf.cuh compiled for the host, driven by tests/test_oprf_host.py: one command per stdin line, one
// result line each.  argv[1] names the curve (256, 384 or 521).  Hex strings; "-" is the empty string.
//   scmul|scadd|scsub a b    scinv a    -> the scalar result mod n (plain, big-endian)
//   widen s / widep s        -> the kL-byte string s mod n / mod p
//   decode e                 -> "1 x y" or "0"
//   xmd N dst msg            -> expand_message_xmd
//   h2c dst msg              -> u0 u1 Q0x Q0y Q1x Q1y Px Py
//   derive mode seed info    -> sk pk
//   evaluate mode sk r info e_1 .. e_m  -> status ev_1 .. ev_m proof ("-" in mode 0)
//   full mode sk info input  -> status output
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../circl_b200/csrc/oprf.cuh"
#include "../../circl_b200/csrc/p256.cuh"
#include "../../circl_b200/csrc/p384.cuh"
#include "../../circl_b200/csrc/p521.cuh"

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

template <class C>
struct Run {
  static constexpr int kW = C::kW, NB = C::kBytes, Ne = oprf::kNe<C>;
  std::vector<uint32_t> table;
  Run() : table(nistp::kTableWords<C>) { nistp::build_base_table<C>(table.data()); }

  std::string fe_hex(const nistp::Fe<C>& plain) {
    uint8_t b[NB];
    nistp::words_to_be<C>(b, plain.v, ~0u);
    return hex(b, NB);
  }
  oprf::Sc<C> sc(const std::string& h) {
    Bytes b = unhex(h);
    uint32_t k[kW];
    nistp::words_from_be<C>(k, b.data());
    oprf::Sc<C> s;
    oprf::sc_to_mont(s, k);
    return s;
  }
  std::string sc_hex(const oprf::Sc<C>& s) {
    uint8_t b[NB];
    oprf::scalar_out(b, s, ~0u);
    return hex(b, NB);
  }
  std::string pt_hex(const nistp::Pt<C>& P) {
    nistp::Fe<C> x, y;
    nistp::pt_to_affine(x, y, P);
    return fe_hex(x) + " " + fe_hex(y);
  }

  std::string line(std::istringstream& in) {
    std::string op;
    in >> op;
    if (op == "scmul" || op == "scadd" || op == "scsub") {
      std::string a, b;
      in >> a >> b;
      oprf::Sc<C> x = sc(a), y = sc(b), r;
      if (op == "scmul") oprf::sc_mul(r, x, y);
      if (op == "scadd") oprf::sc_add(r, x, y);
      if (op == "scsub") oprf::sc_sub(r, x, y);
      return sc_hex(r);
    }
    if (op == "scinv") {
      std::string a;
      in >> a;
      oprf::Sc<C> r;
      oprf::sc_invert(r, sc(a));
      return sc_hex(r);
    }
    if (op == "widen" || op == "widep") {
      std::string a;
      in >> a;
      Bytes b = unhex(a);
      if (op == "widen") {
        oprf::Sc<C> r;
        oprf::sc_from_wide(r, b.data());
        return sc_hex(r);
      }
      nistp::Fe<C> plain, mont;
      oprf::fe_from_wide(plain, mont, b.data());
      return fe_hex(plain);
    }
    if (op == "decode") {
      std::string a;
      in >> a;
      Bytes b = unhex(a);
      nistp::Aff<C> A;
      if (!oprf::decode(A, b.data())) return "0";
      nistp::Fe<C> x, y;
      nistp::fe_from_mont(x, A.x);
      nistp::fe_from_mont(y, A.y);
      return "1 " + fe_hex(x) + " " + fe_hex(y);
    }
    if (op == "xmd") {
      int N;
      std::string d, m;
      in >> N >> d >> m;
      Bytes dst = unhex(d), msg = unhex(m), out(N);
      oprf::expand_xmd<C>(out.data(), N, oprf::Cat<1>{{{msg.data(), (int)msg.size()}}}, dst.data(), (int)dst.size());
      return hex(out.data(), N);
    }
    if (op == "h2c") {
      std::string d, m;
      in >> d >> m;
      Bytes dst = unhex(d), msg = unhex(m);
      nistp::Pt<C> P, Q[2];
      nistp::Fe<C> u[2];
      oprf::hash_to_group<C>(P, oprf::Cat<1>{{{msg.data(), (int)msg.size()}}}, dst.data(), (int)dst.size(), u, Q);
      return fe_hex(u[0]) + " " + fe_hex(u[1]) + " " + pt_hex(Q[0]) + " " + pt_hex(Q[1]) + " " + pt_hex(P);
    }
    int mode;
    in >> mode;
    uint8_t ctx[24];
    const int clen = oprf::context<C>(ctx, mode);
    if (op == "derive") {
      std::string s, i;
      in >> s >> i;
      Bytes seed = unhex(s), info = unhex(i);
      uint8_t sk[NB], pk[Ne];
      oprf::derive_key<C>(sk, pk, seed.data(), info.data(), (int)info.size(), table.data(), ctx, clen);
      return hex(sk, NB) + " " + hex(pk, Ne);
    }
    std::string sk_h, a, b;
    in >> sk_h;
    Bytes skb = unhex(sk_h);
    oprf::Sc<C> m_info{};
    if (op == "full") {
      in >> a >> b;
      Bytes info = unhex(a), input = unhex(b);
      if (mode == 2) m_info = info_scalar(info);
      uint32_t kp[kW], ke[kW];
      const uint32_t st = oprf::op_keys<C>(kp, ke, skb.data(), mode, m_info);
      uint8_t out[oprf::kNh<C>];
      oprf::full_evaluate<C>(out, ke, input.data(), (int)input.size(), info.data(), (int)info.size(), mode, ctx, clen,
                             st ? 0u : ~0u);
      return std::to_string(st) + " " + hex(out, sizeof out);
    }
    if (op == "evaluate") {
      std::string r_h, i_h, e;
      in >> r_h >> i_h;
      Bytes rb = unhex(r_h), info = unhex(i_h), bl;
      int m = 0;
      while (in >> e) {
        Bytes x = unhex(e);
        bl.insert(bl.end(), x.begin(), x.end());
        m++;
      }
      if (mode == 2) m_info = info_scalar(info);
      uint32_t kp[kW], ke[kW];
      uint32_t st = oprf::op_keys<C>(kp, ke, skb.data(), mode, m_info);
      Bytes ev(m * Ne);
      for (int j = 0; j < m; j++) st |= oprf::eval_element<C>(ev.data() + j * Ne, bl.data() + j * Ne, ke);
      std::string res;
      uint8_t proof[2 * NB];
      if (mode != 0) {
        uint8_t Y[Ne];
        nistp::Pt<C> P;
        nistp::scalarmult_base(P, kp, table.data());
        oprf::encode(Y, P, ~0u);
        const uint8_t *bs = mode == 2 ? ev.data() : bl.data(), *cs = mode == 2 ? bl.data() : ev.data();
        nistp::Pt<C> M;
        uint32_t dst = 0;
        oprf::composite<C>(M, dst, Y, bs, Ne, cs, Ne, m, ctx, clen);
        nistp::Fe<C> x, y;
        nistp::pt_to_affine(x, y, M);
        uint8_t mxy[2 * NB];
        nistp::words_to_be<C>(mxy, x.v, ~0u);
        nistp::words_to_be<C>(mxy + NB, y.v, ~0u);
        const uint32_t rok = oprf::prove<C>(proof, kp, Y, mxy, rb.data(), table.data(), ctx, clen, ~0u);
        st |= rok ? 0u : 4u;
      }
      res = std::to_string(st);
      for (int j = 0; j < m; j++) res += " " + hex(ev.data() + j * Ne, Ne);
      return res + " " + (mode ? hex(proof, 2 * NB) : std::string("-"));
    }
    return "?";
  }
  oprf::Sc<C> info_scalar(const Bytes& info) {
    uint8_t ctx[24], dst[13 + 24];
    const int clen = oprf::context<C>(ctx, 2);
    for (int i = 0; i < 13; i++) dst[i] = (uint8_t)"HashToScalar-"[i];
    for (int i = 0; i < clen; i++) dst[13 + i] = ctx[i];
    const oprf::Len2 l((int)info.size());
    oprf::Sc<C> s;
    oprf::hash_to_scalar<C>(s, oprf::Cat<3>{{{(const uint8_t*)"Info", 4}, {l.b, 2}, {info.data(), (int)info.size()}}},
                            dst, 13 + clen);
    return s;
  }
};

template <class C>
static int loop() {
  Run<C> r;
  std::string l;
  while (std::getline(std::cin, l)) {
    std::istringstream in(l);
    std::cout << r.line(in) << "\n";
  }
  return 0;
}

int main(int argc, char** argv) {
  const std::string c = argc > 1 ? argv[1] : "";
  if (c == "256") return loop<nistp::P256>();
  if (c == "384") return loop<nistp::P384>();
  if (c == "521") return loop<nistp::P521>();
  return 2;
}
