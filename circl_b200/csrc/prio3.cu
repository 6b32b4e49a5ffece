// Prio3 aggregator (draft-irtf-cfrg-vdaf-14): the reference's vdaf/prio3 PrepInit, PrepSharesToPrep, PrepNext and
// AggregateUpdate for Count, Sum, SumVec, Histogram and MultiHotCountVec, batched on the device.  The arithmetic is
// prio3.cuh; every kernel is one thread per report (or per output element), instantiated on the field only, so any
// circuit parameters run without a rebuild:
//   PrepInit          prio3_init_kernel<F>    XOF expansions, Query into a per-report work area of
//                                             prio3::work_elems() field elements
//   PrepSharesToPrep  prio3_decide_kernel<F>  sum of the verifier shares, Decide, the joint-rand seed
//   PrepNext          prio3_next_kernel       the joint-rand seed check, the out share
//   Aggregate         prio3_sum_kernel<F>     partial sums of the out shares over row slices, then
//                     prio3_fold_kernel<F>    the slices into the accumulator
// Timed under the prio3 profiling class.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"
#include "prio3.cuh"

namespace cb200 {
namespace prio3k {

using namespace prio3;

struct Key {
  uint8_t b[32];
};

template <class F>
__global__ void __launch_bounds__(128) prio3_init_kernel(Cfg c, Key vk, uint32_t agg, const uint8_t* __restrict__ nonces,
                                                         const uint8_t* __restrict__ pub, size_t pub_stride,
                                                         const uint8_t* __restrict__ in, size_t in_stride,
                                                         uint8_t* __restrict__ state, size_t state_stride,
                                                         uint8_t* __restrict__ share, size_t share_stride,
                                                         uint8_t* __restrict__ status, Fe<F>* __restrict__ work, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t *s = state + i * state_stride, *h = share + i * share_stride;
  const uint32_t st = prep_init<F>(c, vk.b, agg, nonces + i * kNonce, pub + i * pub_stride, in + i * in_stride, s, h,
                                   work + i * c.work);
  if (st) {
    for (size_t j = 0; j < state_stride; j++) s[j] = 0;
    for (size_t j = 0; j < share_stride; j++) h[j] = 0;
  }
  status[i] = (uint8_t)st;
}

template <class F>
__global__ void __launch_bounds__(128) prio3_decide_kernel(Cfg c, const uint8_t* __restrict__ shares, size_t ps,
                                                           uint8_t* __restrict__ msg, size_t msg_len,
                                                           uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t* m = msg + i * msg_len;
  const uint32_t st = prep_shares_to_prep<F>(c, shares + i * c.shares * ps, ps, m);
  if (st)
    for (size_t j = 0; j < msg_len; j++) m[j] = 0;
  status[i] = (uint8_t)st;
}

__global__ void __launch_bounds__(128) prio3_next_kernel(const uint8_t* __restrict__ states, size_t state_len,
                                                         const uint8_t* __restrict__ msgs, size_t msg_len,
                                                         uint8_t* __restrict__ out, size_t out_len,
                                                         uint8_t* __restrict__ status, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* s = states + i * state_len;
  uint8_t diff = 0;
  for (size_t j = 0; j < msg_len; j++) diff |= s[out_len + j] ^ msgs[i * msg_len + j];
  const uint8_t mask = diff ? 0 : 0xff;
  for (size_t j = 0; j < out_len; j++) out[i * out_len + j] = s[j] & mask;
  status[i] = diff ? (uint8_t)kErrJointRand : 0;
}

// raw little-endian limbs, reduced once (an out share element is canonical; a string >= p counts as itself - p)
template <class F>
__device__ __forceinline__ Fe<F> load_raw(const uint8_t* in) {
  uint64_t t[F::N];
  for (int i = 0; i < F::N; i++) {
    uint64_t w = 0;
    for (int j = 0; j < 8; j++) w |= (uint64_t)in[8 * i + j] << (8 * j);
    t[i] = w;
  }
  return reduce_once<F>(t, 0);
}

// part[s][e] = sum of element e over rows s, s + S, s + 2S, ... whose status is 0
template <class F>
__global__ void __launch_bounds__(128) prio3_sum_kernel(const uint8_t* __restrict__ rows, size_t len,
                                                        const uint8_t* __restrict__ status, size_t n, Fe<F>* part) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y, S = gridDim.y;
  if (e >= len) return;
  Fe<F> acc = zero<F>();
  for (size_t r = s; r < n; r += S)
    if (!status || !status[r]) acc = add<F>(acc, load_raw<F>(rows + (r * len + e) * F::kBytes));
  part[s * len + e] = acc;
}

// acc[e] += sum_s part[s][e]
template <class F>
__global__ void __launch_bounds__(128) prio3_fold_kernel(const Fe<F>* part, size_t S, size_t len, Fe<F>* acc) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= len) return;
  Fe<F> a = acc[e];
  for (size_t s = 0; s < S; s++) a = add<F>(a, part[s * len + e]);
  acc[e] = a;
}

static inline unsigned blocks(size_t units, size_t per) { return (unsigned)((units + per - 1) / per); }

// ---------------------------------------------------------------- host side
// Largest work area of one report: 64 MiB (a Histogram of length 2^22, or a Lagrange domain of 2^21 Field128 points).
constexpr uint64_t kMaxWork = 64ull << 20;
// Reports per launch: the work areas of one launch stay within 1 GiB.
constexpr uint64_t kLaunchWork = 1ull << 30;

static int bad(const char* fn, const char* what) {
  set_error("%s: %s", fn, what);
  return CB200_ERR_ARG;
}

// The configuration as the reference's constructors (New) validate it, and the lengths of its FLP.
static int plan(const char* fn, const cb200_prio3_config* k, Cfg* c, cb200_prio3_sizes* z) {
  if (!k) return bad(fn, "null config");
  if (k->num_shares < 2 || k->num_shares > 255) return bad(fn, "invalid numshares (ErrNumShares)");
  if (k->context_len > 65535 - 8) return bad(fn, "invalid context length (ErrContextSize)");
  if (k->context_len && !k->context) return bad(fn, "null context");
  *c = Cfg{};
  c->kind = k->kind;
  c->shares = k->num_shares;
  c->ctxlen = (uint32_t)k->context_len;
  const uint64_t maxu = 1ull << 40;  // beyond any domain the work-area bound admits; keeps the products below exact
  uint64_t calls = 0, meas = 0, out = 0, evo = 0, arity = 0, jr = 0;
  auto bitlen = [](uint64_t v) {
    int b = 0;
    while (v >> b) b++;
    return (uint64_t)b;
  };
  switch (k->kind) {
    case CB200_PRIO3_COUNT:
      calls = meas = out = evo = 1;
      arity = 2;
      break;
    case CB200_PRIO3_SUM:
      if (k->max_measurement >= 1ull << 63) return bad(fn, "max measurement must be less than 2^63");
      c->bits = (uint32_t)bitlen(k->max_measurement);
      c->offset = ((1ull << c->bits) - 1) - k->max_measurement;
      calls = meas = 2 * c->bits;
      out = 1;
      evo = 2 * c->bits + 1;
      arity = 1;
      break;
    case CB200_PRIO3_SUMVEC:
      if (k->length == 0) return bad(fn, "length cannot be zero");
      if (k->bits == 0 || k->bits > 64) return bad(fn, "bits must be between 1 and 64");
      if (k->chunk_length == 0) return bad(fn, "chunk length cannot be zero");
      if (k->length > maxu || k->chunk_length > maxu) return bad(fn, "work area too large");
      meas = k->length * k->bits;
      out = k->length;
      evo = 1;
      c->bits = (uint32_t)k->bits;
      break;
    case CB200_PRIO3_HISTOGRAM:
      if (k->length == 0) return bad(fn, "length cannot be zero");
      if (k->chunk_length == 0) return bad(fn, "chunk length cannot be zero");
      if (k->length > maxu || k->chunk_length > maxu) return bad(fn, "work area too large");
      meas = out = k->length;
      evo = 2;
      break;
    case CB200_PRIO3_MULTIHOT:
      if (k->length == 0) return bad(fn, "length cannot be zero");
      if (k->max_weight > k->length) return bad(fn, "maxWeight cannot be greater than length");
      if (k->chunk_length == 0) return bad(fn, "chunkLength cannot be zero");
      if (k->length > maxu || k->chunk_length > maxu) return bad(fn, "work area too large");
      // ErrFieldSize (p - offset <= length) cannot hold for a length below 2^40
      c->bits = (uint32_t)bitlen(k->max_weight);
      c->offset = ((1ull << c->bits) - 1) - k->max_weight;
      meas = k->length + c->bits;
      out = k->length;
      evo = 2;
      break;
    default:
      return bad(fn, "unknown kind");
  }
  if (k->kind >= CB200_PRIO3_SUMVEC) {
    calls = (meas + k->chunk_length - 1) / k->chunk_length;
    arity = 2 * k->chunk_length;
    jr = calls;
    c->chunk = (uint32_t)k->chunk_length;
    c->length = (uint32_t)k->length;
  }
  uint64_t p = 1;
  int log2p = 0;
  while (p < 1 + calls) p <<= 1, log2p++;
  const uint64_t B = k->kind <= CB200_PRIO3_SUM ? 8 : 16;
  const uint64_t proof = arity + 1 + 2 * (p - 1);
  // the bound is checked on the 64-bit lengths, before they are narrowed into Cfg
  const uint64_t work = meas + proof + jr + evo + 1 + 2 * p + arity;
  if (work * B > kMaxWork) return bad(fn, "work area of one report over 64 MiB");
  c->meas_len = (uint32_t)meas;
  c->out_len = (uint32_t)out;
  c->eval_out_len = (uint32_t)evo;
  c->proof_len = (uint32_t)proof;
  c->verifier_len = (uint32_t)(2 + arity);
  c->jr_len = (uint32_t)jr;
  c->arity = (uint32_t)arity;
  c->calls = (uint32_t)calls;
  c->log2p = (uint32_t)log2p;
  c->work = work_elems(*c);
  const uint64_t J = jr ? kSeed : 0;
  z->input_share_leader = B * (meas + proof) + J;
  z->input_share_helper = kSeed + J;
  z->public_share = jr ? (uint64_t)kSeed * c->shares : 0;
  z->prep_share = B * (2 + arity) + J;
  z->prep_msg = J;
  z->prep_state = B * out + J;
  z->out_share = z->agg_share = B * out;
  return 0;
}

static bool is_f64(const Cfg& c) { return c.kind <= kSum; }

// device copy of the context string in the call's level-1 area, with room for `extra` more bytes after it
static int stage_ctx(const cb200_prio3_config* k, int slot, size_t extra, Arena* A, Cfg* c, cudaStream_t st) {
  int rc = arena(slot, k->context_len + extra + 4096, A);
  if (rc) return rc;
  c->ctx = nullptr;
  if (k->context_len) {
    uint8_t* d = A->take(k->context_len);
    CB200_CUDA(cudaMemcpyAsync(d, k->context, k->context_len, cudaMemcpyHostToDevice, st));
    c->ctx = d;
  }
  return 0;
}

template <class F>
static void launch_init(const Cfg& c, const Key& vk, uint32_t agg, const Rows& r, size_t cnt, size_t per, Fe<F>* work,
                        cudaStream_t st) {
  KernelScope ks(KID_PRIO3, st);
  for (size_t f = 0; f < cnt; f += per) {
    const size_t m = std::min(per, cnt - f);
    prio3_init_kernel<F><<<blocks(m, 128), 128, 0, st>>>(
        c, vk, agg, r[0].p + f * r[0].stride, r[1].p ? r[1].p + f * r[1].stride : nullptr, r[1].stride,
        r[2].p + f * r[2].stride, r[2].stride, r[3].p + f * r[3].stride, r[3].stride, r[4].p + f * r[4].stride,
        r[4].stride, r[5].p + f, work, m);
  }
}

template <class F>
static int sum_rows(const uint8_t* rows, const uint8_t* status, size_t n, size_t len, Fe<F>* part, Fe<F>* acc,
                    cudaStream_t st) {
  const size_t S = std::min<size_t>(n, 256);
  KernelScope ks(KID_PRIO3, st);
  prio3_sum_kernel<F><<<dim3(blocks(len, 128), (unsigned)S), 128, 0, st>>>(rows, len, status, n, part);
  prio3_fold_kernel<F><<<blocks(len, 128), 128, 0, st>>>(part, S, len, acc);
  CB200_CUDA(cudaGetLastError());
  return 0;
}

// Aggregate: on device buffers, one pass on the caller's stream; on host buffers, one range per GPU staged in chunks,
// each GPU's partial sum copied back and added on the host.
template <class F>
static int aggregate(const char* fn, size_t len, const uint8_t* out_shares, const uint8_t* status, uint8_t* agg,
                     size_t n, bool dev) {
  const size_t row = len * F::kBytes;
  if (dev) {
    DeviceCall call(out_shares);
    if (call.rc) return call.rc;
    Arena A;
    const size_t S = std::min<size_t>(n, 256);  // partial rows: sum_rows uses min(rows, 256) slices
    int rc = arena(kDevSlot, (S + 1) * row + 4096, &A);
    if (rc) return rc;
    Fe<F>*part = (Fe<F>*)A.take(S * row), *acc = (Fe<F>*)A.take(row);
    CB200_CUDA(cudaMemsetAsync(acc, 0, row, call.st));
    const size_t chunk = std::max<size_t>(1, (1u << 30) / row);
    for (size_t f = 0; f < n; f += chunk) {
      rc = sum_rows<F>(out_shares + f * row, status ? status + f : nullptr, std::min(chunk, n - f), len, part, acc,
                       call.st);
      if (rc) return rc;
    }
    CB200_CUDA(cudaMemcpyAsync(agg, acc, row, cudaMemcpyDeviceToDevice, call.st));
    return 0;
  }
  std::vector<Fe<F>> total(len, zero<F>());
  std::mutex mu;
  const size_t chunk = std::max<size_t>(1, std::min<size_t>(1u << 16, (64u << 20) / row));
  int rc = for_each_shard(n, 1u << 14, [&](size_t f0, size_t sn) -> int {
    Dev& d = ctx();
    cudaStream_t st = d.pipe[0];
    const size_t img = chunk * row, sbytes = (chunk + 255) & ~(size_t)255, pbytes = std::min<size_t>(std::min(chunk, sn), 256) * row;
    int rc2 = ensure_scratch(0, img + sbytes + pbytes + row);
    if (rc2) return rc2;
    uint8_t* base = (uint8_t*)d.scratch[0];
    uint8_t *drows = base, *dstat = base + img;
    Fe<F>*part = (Fe<F>*)(base + img + sbytes), *acc = (Fe<F>*)(base + img + sbytes + pbytes);
    CB200_CUDA(cudaMemsetAsync(acc, 0, row, st));
    for (size_t f = f0; f < f0 + sn; f += chunk) {
      const size_t m = std::min(chunk, f0 + sn - f);
      CB200_CUDA(cudaMemcpyAsync(drows, out_shares + f * row, m * row, cudaMemcpyHostToDevice, st));
      if (status) CB200_CUDA(cudaMemcpyAsync(dstat, status + f, m, cudaMemcpyHostToDevice, st));
      rc2 = sum_rows<F>(drows, status ? dstat : nullptr, m, len, part, acc, st);
      if (rc2) return rc2;
      CB200_CUDA(cudaStreamSynchronize(st));  // the image is reused by the next chunk
    }
    std::vector<Fe<F>> mine(len);
    CB200_CUDA(cudaMemcpyAsync(mine.data(), acc, row, cudaMemcpyDeviceToHost, st));
    CB200_CUDA(cudaStreamSynchronize(st));
    std::lock_guard<std::mutex> g(mu);
    for (size_t e = 0; e < len; e++) total[e] = add<F>(total[e], mine[e]);
    return 0;
  });
  if (rc) return rc;
  memcpy(agg, total.data(), row);  // limbs are little-endian: the canonical encoding
  return 0;
}

}  // namespace prio3k
}  // namespace cb200

using namespace cb200;
using namespace cb200::prio3k;

extern "C" {

int cb200_prio3_get_sizes(const cb200_prio3_config* cfg, cb200_prio3_sizes* out) {
  Cfg c;
  cb200_prio3_sizes z;
  int rc = plan("cb200_prio3_get_sizes", cfg, &c, &z);
  if (rc) return rc;
  if (!out) return bad("cb200_prio3_get_sizes", "null pointer");
  *out = z;
  return 0;
}

int cb200_prio3_prep_init(const cb200_prio3_config* cfg, const uint8_t* verify_key, uint32_t agg_id,
                          const uint8_t* nonces, const uint8_t* public_shares, const uint8_t* input_shares,
                          uint8_t* prep_states, uint8_t* prep_shares, uint8_t* status, size_t n) {
  const char* fn = "cb200_prio3_prep_init";
  Cfg c;
  cb200_prio3_sizes z;
  int rc = plan(fn, cfg, &c, &z);
  if (rc) return rc;
  if (agg_id >= c.shares) return bad(fn, "invalid aggregation ID (ErrAggID)");
  if (!verify_key || !nonces || !input_shares || !prep_states || !prep_shares || !status ||
      (z.public_share && !public_shares))
    return bad(fn, "null pointer");
  if ((rc = require_ready())) return rc;
  if (n == 0) return 0;
  Key vk;
  memcpy(vk.b, verify_key, 32);
  const size_t in = agg_id ? z.input_share_helper : z.input_share_leader;
  const size_t B = is_f64(c) ? 8 : 16, work = c.work * B;
  const size_t per = std::max<uint64_t>(1, std::min<uint64_t>(1u << 15, kLaunchWork / work));
  const uint8_t* pub = z.public_share ? public_shares : nullptr;
  Batch b{fn, n, prep_states, per, std::max<size_t>(1, per / 8),
          {{nonces, kNonce, kNonce, kIn}, {pub, z.public_share, z.public_share, kIn}, {input_shares, in, in, kIn},
           {prep_states, z.prep_state, z.prep_state, kOut}, {prep_shares, z.prep_share, z.prep_share, kOut},
           {status, 1, 1, kStatus}},
          {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    Cfg cc = c;
    const size_t m = std::min(cnt, per);
    int rc2 = stage_ctx(cfg, slot, m * work + 256, &A, &cc, st);
    if (rc2) return rc2;
    void* w = A.take(m * work);
    if (is_f64(cc))
      launch_init<F64>(cc, vk, agg_id, r, cnt, per, (Fe<F64>*)w, st);
    else
      launch_init<F128>(cc, vk, agg_id, r, cnt, per, (Fe<F128>*)w, st);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

int cb200_prio3_prep_shares_to_prep(const cb200_prio3_config* cfg, const uint8_t* prep_shares, uint8_t* prep_msgs,
                                    uint8_t* status, size_t n) {
  const char* fn = "cb200_prio3_prep_shares_to_prep";
  Cfg c;
  cb200_prio3_sizes z;
  int rc = plan(fn, cfg, &c, &z);
  if (rc) return rc;
  if (!prep_shares || !status || (z.prep_msg && !prep_msgs)) return bad(fn, "null pointer");
  if ((rc = require_ready())) return rc;
  if (n == 0) return 0;
  const size_t row = c.shares * z.prep_share;
  const size_t per = std::max<size_t>(1, std::min<size_t>(1u << 16, (256u << 20) / row));
  uint8_t* msgs = z.prep_msg ? prep_msgs : nullptr;
  Batch b{fn, n, prep_shares, per, std::max<size_t>(1, per / 8),
          {{prep_shares, row, row, kIn}, {msgs, z.prep_msg, z.prep_msg, kOut}, {status, 1, 1, kStatus}}, {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int slot) -> int {
    Arena A;
    Cfg cc = c;
    int rc2 = stage_ctx(cfg, slot, 0, &A, &cc, st);
    if (rc2) return rc2;
    KernelScope ks(KID_PRIO3, st);
    if (is_f64(cc))
      prio3_decide_kernel<F64><<<blocks(cnt, 128), 128, 0, st>>>(cc, r[0].p, z.prep_share, r[1].p, z.prep_msg, r[2].p,
                                                                 cnt);
    else
      prio3_decide_kernel<F128><<<blocks(cnt, 128), 128, 0, st>>>(cc, r[0].p, z.prep_share, r[1].p, z.prep_msg,
                                                                  r[2].p, cnt);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

int cb200_prio3_prep_next(const cb200_prio3_config* cfg, const uint8_t* prep_states, const uint8_t* prep_msgs,
                          uint8_t* out_shares, uint8_t* status, size_t n) {
  const char* fn = "cb200_prio3_prep_next";
  Cfg c;
  cb200_prio3_sizes z;
  int rc = plan(fn, cfg, &c, &z);
  if (rc) return rc;
  if (!prep_states || !out_shares || !status || (z.prep_msg && !prep_msgs)) return bad(fn, "null pointer");
  if ((rc = require_ready())) return rc;
  if (n == 0) return 0;
  const size_t per = std::max<size_t>(1, std::min<size_t>(1u << 16, (256u << 20) / z.prep_state));
  const uint8_t* msgs = z.prep_msg ? prep_msgs : nullptr;
  Batch b{fn, n, out_shares, per, std::max<size_t>(1, per / 8),
          {{prep_states, z.prep_state, z.prep_state, kIn}, {msgs, z.prep_msg, z.prep_msg, kIn},
           {out_shares, z.out_share, z.out_share, kOut}, {status, 1, 1, kStatus}},
          {}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) -> int {
    KernelScope ks(KID_PRIO3, st);
    prio3_next_kernel<<<blocks(cnt, 128), 128, 0, st>>>(r[0].p, z.prep_state, r[1].p, z.prep_msg, r[2].p, z.out_share,
                                                        r[3].p, cnt);
    CB200_CUDA(cudaGetLastError());
    return 0;
  });
}

int cb200_prio3_aggregate(const cb200_prio3_config* cfg, const uint8_t* out_shares, const uint8_t* status,
                          uint8_t* agg_share, size_t n) {
  const char* fn = "cb200_prio3_aggregate";
  Cfg c;
  cb200_prio3_sizes z;
  int rc = plan(fn, cfg, &c, &z);
  if (rc) return rc;
  if (!out_shares || !agg_share) return bad(fn, "null pointer");
  if ((rc = require_ready())) return rc;
  const bool dev = is_device_ptr(agg_share);
  if (is_device_ptr(out_shares) != dev || (status && is_device_ptr(status) != dev))
    return bad(fn, "mixed host/device pointers");
  if (n == 0) {
    if (dev) {
      DeviceCall call(agg_share);
      if (call.rc) return call.rc;
      CB200_CUDA(cudaMemsetAsync(agg_share, 0, z.agg_share, call.st));
    } else {
      memset(agg_share, 0, z.agg_share);
    }
    return 0;
  }
  if (is_f64(c)) return aggregate<F64>(fn, c.out_len, out_shares, status, agg_share, n, dev);
  return aggregate<F128>(fn, c.out_len, out_shares, status, agg_share, n, dev);
}

}  // extern "C"
