// circl_b200/csrc/prio3.cuh compiled for the host (g++), driven line by line from tests/test_prio3_host.py:
//   fmul|fadd|fsub|finv <bits> <a> <b>   field operations on canonical hex (big-endian) values -> result
//   ntt <bits> <logn> <hex elements...>  forward NTT then the inverse (NTT, reverse [1:], times 2^-logn) -> both
//   init <cfg...> <ctx> <vk> <agg> <nonce> <pub> <in>  PrepInit -> status state share
//   decide <cfg...> <ctx> <rows>         PrepSharesToPrep -> status msg
//   query <cfg...> <ctx> <t> <meas || proof> <jr> <qr>  Query at a given t (hex element strings as on the wire)
//                                        -> status verifier
// <cfg...> is kind shares meas_len out_len eval_out_len proof_len verifier_len jr_len arity calls chunk bits length
// log2p offset; "-" stands for an empty hex string.
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include <cstdint>
namespace cb200 {
namespace keccak {
// Keccak-p[1600] rounds first_round..23 (FIPS 202), plain C++
void f1600(uint64_t (&a)[25], int first_round) {
  static const int rho[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
  uint64_t rc[24];
  uint32_t lfsr = 1;
  for (int r = 0; r < 24; r++) {
    uint64_t c = 0;
    for (int j = 0; j < 7; j++) {
      if (lfsr & 1) c ^= 1ULL << ((1u << j) - 1);
      lfsr = ((lfsr << 1) ^ ((lfsr & 0x80) ? 0x171u : 0u)) & 0xffu;
    }
    rc[r] = c;
  }
  for (int r = first_round; r < 24; r++) {
    uint64_t c[5], b[25];
    for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
    for (int i = 0; i < 25; i++) {
      const int x = i % 5, y = i / 5;
      const uint64_t v = a[i] ^ c[(x + 4) % 5] ^ ((c[(x + 1) % 5] << 1) | (c[(x + 1) % 5] >> 63));
      b[y + 5 * ((2 * x + 3 * y) % 5)] = rho[i] ? (v << rho[i]) | (v >> (64 - rho[i])) : v;
    }
    for (int y = 0; y < 25; y += 5)
      for (int x = 0; x < 5; x++) a[y + x] = b[y + x] ^ (~b[y + (x + 1) % 5] & b[y + (x + 2) % 5]);
    a[0] ^= rc[r];
  }
}
}  // namespace keccak
}  // namespace cb200

#include "../../circl_b200/csrc/prio3.cuh"

using namespace cb200::prio3;

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> v;
  if (s == "-") return v;
  for (size_t i = 0; i + 1 < s.size(); i += 2) v.push_back((uint8_t)std::stoi(s.substr(i, 2), nullptr, 16));
  return v;
}
static std::string hex(const uint8_t* b, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; i++) s += d[b[i] >> 4], s += d[b[i] & 15];
  return n ? s : "-";
}
// canonical big-endian hex <-> element (Montgomery form)
template <class F>
static Fe<F> elt(const std::string& s) {
  std::vector<uint8_t> be = unhex(s), le(F::kBytes);
  for (int i = 0; i < F::kBytes; i++) le[i] = be[F::kBytes - 1 - i];
  Fe<F> a;
  load<F>(a, le.data());
  return a;
}
template <class F>
static std::string str(const Fe<F>& a) {
  uint8_t le[F::kBytes], be[F::kBytes];
  store<F>(le, a);
  for (int i = 0; i < F::kBytes; i++) be[i] = le[F::kBytes - 1 - i];
  return hex(be, F::kBytes);
}

static Cfg read_cfg(std::istringstream& in, std::vector<uint8_t>& ctx) {
  Cfg c{};
  in >> c.kind >> c.shares >> c.meas_len >> c.out_len >> c.eval_out_len >> c.proof_len >> c.verifier_len >> c.jr_len >>
      c.arity >> c.calls >> c.chunk >> c.bits >> c.length >> c.log2p >> c.offset;
  std::string s;
  in >> s;
  ctx = unhex(s);
  c.ctx = ctx.data();
  c.ctxlen = (uint32_t)ctx.size();
  c.work = work_elems(c);
  return c;
}

template <class F>
static void field_op(const std::string& op, std::istringstream& in) {
  std::string a, b;
  in >> a >> b;
  const Fe<F> x = elt<F>(a), y = elt<F>(b);
  Fe<F> r = op == "fmul" ? mul<F>(x, y) : op == "fadd" ? add<F>(x, y) : op == "fsub" ? sub<F>(x, y) : inv<F>(x);
  std::cout << str<F>(r) << "\n";
}

template <class F>
static void ntt_op(std::istringstream& in) {
  int logn;
  in >> logn;
  std::vector<Fe<F>> v(1u << logn);
  for (auto& e : v) {
    std::string s;
    in >> s;
    e = elt<F>(s);
  }
  ntt<F>(v.data(), logn);
  std::string out;
  for (auto& e : v) out += str<F>(e) + " ";
  std::vector<Fe<F>> w = v;
  ntt<F>(w.data(), logn);
  const Fe<F> s = inv_two_n<F>(logn);
  for (size_t k = 0; k < w.size(); k++) out += str<F>(mul<F>(w[k ? w.size() - k : 0], s)) + (k + 1 < w.size() ? " " : "");
  std::cout << out << "\n";
}

template <class F>
static void init_op(const Cfg& c, std::istringstream& in) {
  std::string s;
  std::vector<uint8_t> f[5];
  uint32_t agg;
  in >> s;
  f[0] = unhex(s);
  in >> agg;
  for (int i = 1; i < 4; i++) in >> s, f[i] = unhex(s);
  std::vector<Fe<F>> work(c.work);
  std::vector<uint8_t> state(F::kBytes * c.out_len + (c.jr_len ? kSeed : 0)),
      share(F::kBytes * c.verifier_len + (c.jr_len ? kSeed : 0));
  const uint32_t st = prep_init<F>(c, f[0].data(), agg, f[1].data(), f[2].data(), f[3].data(), state.data(),
                                   share.data(), work.data());
  std::cout << st << " " << (st ? "-" : hex(state.data(), state.size())) << " "
            << (st ? "-" : hex(share.data(), share.size())) << "\n";
}

template <class F>
static void decide_op(const Cfg& c, std::istringstream& in) {
  std::string s;
  in >> s;
  std::vector<uint8_t> rows = unhex(s);
  const size_t ps = rows.size() / c.shares;
  std::vector<uint8_t> msg(c.jr_len ? kSeed : 0);
  const uint32_t st = prep_shares_to_prep<F>(c, rows.data(), ps, msg.data());
  std::cout << st << " " << (st ? "-" : hex(msg.data(), msg.size())) << "\n";
}

template <class F>
static std::vector<Fe<F>> elts(const std::string& s) {
  const std::vector<uint8_t> b = unhex(s);
  std::vector<Fe<F>> v(b.size() / F::kBytes);
  for (size_t i = 0; i < v.size(); i++) load<F>(v[i], b.data() + F::kBytes * i);
  return v;
}

template <class F>
static void query_op(const Cfg& c, std::istringstream& in) {
  std::string ts, ms, js, qs;
  in >> ts >> ms >> js >> qs;
  const std::vector<Fe<F>> t = elts<F>(ts), mp = elts<F>(ms), jr = elts<F>(js), qr = elts<F>(qs);
  const uint32_t p = 1u << c.log2p;
  std::vector<Fe<F>> w(2 * p + c.arity + 1);
  std::vector<uint8_t> out(F::kBytes * c.verifier_len);
  const uint32_t st = query<F>(c, t[0], mp.data(), mp.data() + c.meas_len, jr.data(), qr.data(), w.data(),
                               w.data() + p, w.data() + 2 * p, out.data());
  std::cout << st << " " << (st ? "-" : hex(out.data(), out.size())) << "\n";
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    in >> op;
    if (op[0] == 'f') {
      int bits;
      in >> bits;
      if (bits == 64) field_op<F64>(op, in);
      else field_op<F128>(op, in);
    } else if (op == "ntt") {
      int bits;
      in >> bits;
      if (bits == 64) ntt_op<F64>(in);
      else ntt_op<F128>(in);
    } else {
      std::vector<uint8_t> ctx;
      const Cfg c = read_cfg(in, ctx);
      const bool f64 = c.kind <= kSum;
      if (op == "init") {
        if (f64) init_op<F64>(c, in);
        else init_op<F128>(c, in);
      } else if (op == "query") {
        if (f64) query_op<F64>(c, in);
        else query_op<F128>(c, in);
      } else {
        if (f64) decide_op<F64>(c, in);
        else decide_op<F128>(c, in);
      }
    }
    std::cout.flush();
  }
  return 0;
}
