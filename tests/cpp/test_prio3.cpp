// The C++ circl::prio3 mirror (include/circl_b200.hpp), driven line by line from tests/test_cpp_prio3.py.  Every line
// starts with the configuration: kind shares max_measurement length bits chunk_length max_weight context, then
//   sizes                                  -> the eight wire sizes, or "ERR <what>" for a refused configuration
//   init <vk> <agg> <nonce> <pub> <in>     PrepInit -> "<status> <state> <share>" (per-report call: the error name)
//   decide <share> ...                     PrepSharesToPrep over the shares -> prep message
//   next <state> <msg>                     PrepNext -> out share
//   unshard <num> <agg share> ...          AggregateUpdate of each agg share into a zero one, then Unshard -> values
// "-" stands for an empty hex string.  Without a device, a call prints "NODEV".
#include <iostream>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "circl_b200.hpp"

using circl::Bytes;
namespace p3 = circl::prio3;

static Bytes unhex(const std::string& s) {
  Bytes v;
  if (s == "-") return v;
  for (size_t i = 0; i + 1 < s.size(); i += 2) v.push_back((uint8_t)std::stoi(s.substr(i, 2), nullptr, 16));
  return v;
}
static std::string hex(const Bytes& b) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (uint8_t x : b) s += d[x >> 4], s += d[x & 15];
  return b.empty() ? "-" : s;
}

static std::unique_ptr<p3::Prio3> make(std::istringstream& in) {
  unsigned kind, shares;
  uint64_t mx, len, bits, chunk, weight;
  std::string ctx;
  in >> kind >> shares >> mx >> len >> bits >> chunk >> weight >> ctx;
  const Bytes c = unhex(ctx);
  switch (kind) {
    case 1: return std::make_unique<p3::Count>(shares, c);
    case 2: return std::make_unique<p3::Sum>(shares, mx, c);
    case 3: return std::make_unique<p3::SumVec>(shares, len, bits, chunk, c);
    case 4: return std::make_unique<p3::Histogram>(shares, len, chunk, c);
    default: return std::make_unique<p3::MultiHotCountVec>(shares, len, weight, chunk, c);
  }
}

int main() {
  bool dev = true;
  try {
    circl::init(0);
  } catch (const circl::Error&) {
    dev = false;
  }
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    in >> op;
    try {
      auto v = make(in);
      if (op == "sizes") {
        const cb200_prio3_sizes& z = v->Params();
        std::cout << z.input_share_leader << " " << z.input_share_helper << " " << z.public_share << " " << z.prep_share
                  << " " << z.prep_msg << " " << z.prep_state << " " << z.out_share << " " << z.agg_share << "\n";
        continue;
      }
      if (!dev) {
        std::cout << "NODEV\n";
        continue;
      }
      std::string a, b, c, d, e;
      if (op == "init") {
        unsigned agg;
        in >> a >> agg >> b >> c >> d;
        Bytes st, sh;
        try {
          v->PrepInit(unhex(a), unhex(b), (uint8_t)agg, unhex(c), unhex(d), &st, &sh);
          std::cout << "0 " << hex(st) << " " << hex(sh) << "\n";
        } catch (const p3::Prio3Error& x) {
          std::cout << (int)x.status << " " << x.what() << "\n";
        }
      } else if (op == "decide") {
        std::vector<Bytes> shares;
        while (in >> a) shares.push_back(unhex(a));
        try {
          const Bytes msg = v->PrepSharesToPrep(shares);  // before any output: it may throw
          std::cout << "0 " << hex(msg) << "\n";
        } catch (const p3::Prio3Error& x) {
          std::cout << (int)x.status << " " << x.what() << "\n";
        }
      } else if (op == "next") {
        in >> a >> b;
        try {
          const Bytes out = v->PrepNext(unhex(a), unhex(b));
          std::cout << "0 " << hex(out) << "\n";
        } catch (const p3::Prio3Error& x) {
          std::cout << (int)x.status << " " << x.what() << "\n";
        }
      } else if (op == "unshard") {
        uint64_t num;
        in >> num;
        std::vector<Bytes> aggs;
        while (in >> a) {
          Bytes s = v->AggregateInit();
          v->AggregateUpdate(&s, unhex(a));
          aggs.push_back(s);
        }
        std::string out;
        for (uint64_t x : v->Unshard(aggs, num)) out += std::to_string(x) + " ";
        std::cout << out << "\n";
      }
    } catch (const std::invalid_argument& x) {
      std::cout << "ERR " << x.what() << "\n";
    } catch (const std::exception& x) {
      std::cout << "EXC " << x.what() << "\n";
    }
    std::cout.flush();
  }
  return 0;
}
