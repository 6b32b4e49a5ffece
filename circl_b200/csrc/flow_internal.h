// Helpers shared by the flows that compose the lattice flows with a curve (hybrid.cu, eddsa.cu, ed448.cu), and the
// host/device dispatch of every batched C entry point (run_batch).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <functional>
#include <initializer_list>
#include <vector>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"

namespace cb200 {

// bump allocator over the level-1 work area of a slot (level 0 belongs to the lattice flows the caller runs)
struct Arena {
  char* base = nullptr;
  size_t off = 0;
  uint8_t* take(size_t bytes) {
    uint8_t* p = (uint8_t*)(base + off);
    off += (bytes + 255) & ~(size_t)255;
    return p;
  }
};
inline int arena(int slot, size_t bytes, Arena* a) {
  void* p = nullptr;
  int rc = ensure_work(kLevel1 + slot, bytes + 4096, &p);
  if (rc) return rc;
  a->base = (char*)p;
  a->off = 0;
  return 0;
}

// 2D device-to-device copy on the call's stream: n rows of `width` bytes
inline int copy2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t n, cudaStream_t st) {
  CB200_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, n, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---------------------------------------------------------------- batched entry points
// Every batched C entry point describes its call as data (Batch) and hands one body to run_batch, which makes the
// routing decision: all buffers on one side, device rules, then either the caller's stream (device buffers) or the
// staging pipeline (host buffers).  body(rows, count, st, slot) sees, per buffer, the pointer and the stride to use:
// for device calls the caller's, for host calls the staged image with stride `unit` (0 for a shared row).
enum Role { kIn, kOut, kInOut, kStatus, kScratch };
struct Arg {
  const void* p;  // caller's buffer; null = absent (an optional buffer)
  size_t unit;    // bytes per operation
  size_t stride;  // caller's bytes between operations; 0 = one row shared by the batch
  // kStatus: per-op status bytes (optional for the caller; always staged and counted on the host path).
  // kScratch: `unit` bytes per op of device area on the host path (unit 0 = none), nothing copied.
  Role role;
};
struct Row {
  uint8_t* p;
  size_t stride;
};
struct Rows {
  std::vector<Row> r;  // one per Arg, in order; absent buffers are {nullptr, 0}
  const uint8_t* msgs = nullptr;
  const uint64_t* msg_off = nullptr;
  const uint8_t* ctx = nullptr;  // device copy of the context string (null if it is empty)
  const Row& operator[](size_t i) const { return r[i]; }
};
struct DevCheck {  // a rule of device-pointer calls only: fmt is the error text, printed with (function name, n)
  bool fails;
  const char* fmt;
};
struct Batch {
  const char* fn;    // name in error texts
  size_t n;
  const void* bind;  // DeviceCall binds the GPU that holds this buffer
  size_t chunk, min_shard;  // host path: staging chunk and smallest shard per GPU
  std::vector<Arg> args;
  std::vector<DevCheck> dev_checks;  // in order; alignment rules among them
  // variable-length messages (the host path then stages chunks on slot 0) and a shared context string, which is
  // always in host memory and at most 255 bytes
  const uint8_t* msgs = nullptr;
  const uint64_t* msg_off = nullptr;
  const uint8_t* ctx = nullptr;
  size_t ctxlen = 0;
  std::function<int()> host;  // replaces the staged host path (the call keeps its own pipeline)
};
struct Counts {  // per-op status bytes of a host-pointer call
  size_t bit0 = 0, bit1 = 0, nonzero = 0;
};
using Body = std::function<int(const Rows& rows, size_t count, cudaStream_t st, int slot)>;

inline bool aligned(std::initializer_list<const void*> ps, std::initializer_list<size_t> strides, uintptr_t a) {
  uintptr_t acc = 0;
  for (const void* p : ps) acc |= (uintptr_t)p;
  for (size_t v : strides) acc |= v;
  return (acc & (a - 1)) == 0;
}

// Host-pointer calls with variable-length messages: one contiguous range per GPU, staged in chunks through scratch
// slot 0 (bodies run with slot 0); the messages of a chunk follow its rows, with offsets rebased to the chunk.
using MsgBody = std::function<int(uint8_t** d, const uint8_t* msgs, const uint64_t* off, size_t cnt, cudaStream_t st)>;
inline int run_msgs(size_t n, const std::vector<Buf>& rows, const uint8_t* msgs, const uint64_t* msg_off, size_t chunk,
                    size_t min_shard, const MsgBody& body) {
  return for_each_shard(n, min_shard, [&](size_t f0, size_t sn) -> int {
    Dev& c = ctx();
    cudaStream_t st = c.pipe[0];
    std::vector<uint64_t> ro;
    for (size_t first = f0; first < f0 + sn; first += chunk) {
      const size_t cnt = std::min(chunk, f0 + sn - first);
      const uint64_t m0 = msg_off[first];
      const size_t mb = (size_t)(msg_off[first + cnt] - m0);
      size_t off = 0;
      auto take = [&](size_t bytes) {
        size_t o = off;
        off += (bytes + 255) & ~(size_t)255;
        return o;
      };
      std::vector<size_t> ro_off(rows.size());
      for (size_t j = 0; j < rows.size(); j++) ro_off[j] = take(rows[j].shared ? rows[j].unit : cnt * rows[j].unit);
      const size_t oMsg = take(mb + 8), oOff = take((cnt + 1) * 8);
      int rc = ensure_scratch(0, off);
      if (rc) return rc;
      char* d = (char*)c.scratch[0];
      std::vector<uint8_t*> dp(rows.size());
      for (size_t j = 0; j < rows.size(); j++) {
        const Buf& r = rows[j];
        const uint8_t* in = (const uint8_t*)r.host_in;
        dp[j] = (uint8_t*)d + ro_off[j];
        if (!in) continue;
        const size_t hs = r.host_stride ? r.host_stride : r.unit;
        if (r.shared)
          CB200_CUDA(cudaMemcpyAsync(dp[j], in, r.unit, cudaMemcpyHostToDevice, st));
        else if (hs == r.unit)
          CB200_CUDA(cudaMemcpyAsync(dp[j], in + first * hs, cnt * r.unit, cudaMemcpyHostToDevice, st));
        else
          CB200_CUDA(cudaMemcpy2DAsync(dp[j], r.unit, in + first * hs, hs, r.unit, cnt, cudaMemcpyHostToDevice, st));
      }
      if (mb) CB200_CUDA(cudaMemcpyAsync(d + oMsg, msgs + m0, mb, cudaMemcpyHostToDevice, st));
      ro.resize(cnt + 1);
      for (size_t i = 0; i <= cnt; i++) ro[i] = msg_off[first + i] - m0;
      CB200_CUDA(cudaMemcpyAsync(d + oOff, ro.data(), (cnt + 1) * 8, cudaMemcpyHostToDevice, st));
      rc = body(dp.data(), (const uint8_t*)d + oMsg, (const uint64_t*)(d + oOff), cnt, st);
      if (rc) return rc;
      for (size_t j = 0; j < rows.size(); j++)
        if (rows[j].host_out) CB200_CUDA(cudaMemcpyAsync((uint8_t*)rows[j].host_out + first * rows[j].unit, dp[j],
                                                         cnt * rows[j].unit, cudaMemcpyDeviceToHost, st));
      CB200_CUDA(cudaStreamSynchronize(st));  // `ro` and the scratch are reused by the next chunk
    }
    return 0;
  });
}

// Runs a batched call described by `b` (the entry point has checked its arguments and returned on n == 0).
// counts (may be null) receives the status-byte counts of a host-pointer call; device-pointer calls leave the status
// bytes to the caller.
inline int run_batch(const Batch& b, const Body& body, Counts* counts = nullptr) {
  bool dev = false, first = true;
  auto same_side = [&](const void* p) {
    if (!p) return true;
    const bool d = is_device_ptr(p);
    if (first) {
      dev = d;
      first = false;
    }
    return d == dev;
  };
  bool same = same_side(b.msgs) && same_side(b.msg_off);
  for (const Arg& a : b.args) same = same && same_side(a.p);
  if (!same) {
    set_error("%s: mixed host/device pointers", b.fn);
    return CB200_ERR_ARG;
  }
  const size_t na = b.args.size();
  if (dev) {
    for (const DevCheck& c : b.dev_checks)
      if (c.fails) {
        set_error(c.fmt, b.fn, b.n);
        return CB200_ERR_ARG;
      }
    DeviceCall call(b.bind);
    if (call.rc) return call.rc;
    Rows rows;
    for (const Arg& a : b.args) rows.r.push_back(Row{(uint8_t*)a.p, a.stride});
    rows.msgs = b.msgs;
    rows.msg_off = b.msg_off;
    if (b.ctxlen) {  // the context string is at most 255 bytes and always a host pointer: stage it
      CB200_CUDA(cudaMemcpyAsync(call.ws->small, b.ctx, b.ctxlen, cudaMemcpyHostToDevice, call.st));
      rows.ctx = (const uint8_t*)call.ws->small;
    }
    return body(rows, b.n, call.st, kDevSlot);
  }
  if (b.host) return b.host();
  // host buffers: bufs[at[i]] is the staged image of args[i]
  std::vector<Buf> bufs;
  std::vector<int> at(na, -1);
  int status = -1;
  uint8_t* user_status = nullptr;
  std::vector<uint8_t> own;  // status bytes of a message call whose caller passed none
  for (size_t i = 0; i < na; i++) {
    const Arg& a = b.args[i];
    Buf f{nullptr, nullptr, a.unit, a.stride == 0, a.stride};
    if (a.role == kIn || a.role == kInOut) f.host_in = a.p;
    if (a.role == kOut || a.role == kInOut) f.host_out = (void*)a.p;
    if (a.role == kStatus) {
      status = (int)bufs.size();
      user_status = (uint8_t*)a.p;
      if (b.msgs) {  // the message path copies the status bytes out like any output
        if (!user_status) {
          own.resize(b.n);
          user_status = own.data();
        }
        f.host_out = user_status;
      }
    } else if (a.role == kScratch ? a.unit == 0 : a.p == nullptr) {
      continue;
    }
    at[i] = (int)bufs.size();
    bufs.push_back(f);
  }
  auto rows_of = [&](uint8_t** d) {
    Rows rows;
    rows.r.assign(na, Row{nullptr, 0});
    for (size_t i = 0; i < na; i++)
      if (at[i] >= 0) rows.r[i] = Row{d[at[i]], bufs[at[i]].shared ? 0 : bufs[at[i]].unit};
    return rows;
  };
  if (!b.msgs) {
    HostCall hc;
    hc.bufs = bufs;
    hc.chunk = b.chunk;
    hc.min_shard = b.min_shard;
    hc.status_buf = status;
    hc.user_status = user_status;
    hc.body = [&](void** d, size_t cnt, size_t, cudaStream_t st, int slot) {
      return body(rows_of((uint8_t**)d), cnt, st, slot);
    };
    int rc = hc.run(b.n);
    if (rc) return rc;
    if (counts) *counts = Counts{hc.bit0, hc.bit1, hc.nonzero};
    return 0;
  }
  const int ictx = (int)bufs.size();
  if (b.ctxlen) bufs.push_back(Buf{b.ctx, nullptr, b.ctxlen, true, 0});
  int rc = run_msgs(b.n, bufs, b.msgs, b.msg_off, b.chunk, b.min_shard,
                    [&](uint8_t** d, const uint8_t* m, const uint64_t* o, size_t cnt, cudaStream_t st) {
                      Rows rows = rows_of(d);
                      rows.msgs = m;
                      rows.msg_off = o;
                      if (b.ctxlen) rows.ctx = d[ictx];
                      return body(rows, cnt, st, 0);
                    });
  if (rc) return rc;
  if (counts && status >= 0) {
    Counts c;
    for (size_t i = 0; i < b.n; i++) {
      c.bit0 += (user_status[i] & 1) != 0;
      c.bit1 += (user_status[i] & 2) != 0;
      c.nonzero += user_status[i] != 0;
    }
    *counts = c;
  }
  return 0;
}

// the signature families' error for status bytes left set: the 576-attempt cap of the Dilithium signing loop
inline int sign_attempts_result(const char* fn, size_t bad, size_t n) {
  if (!bad) return 0;
  set_error("%s: %zu of %zu signatures exhausted 576 attempts", fn, bad, n);
  return CB200_ERR_SIGN_ATTEMPTS;
}

namespace hybrid {
// out[i] = SHAKE256(in[i] (inlen <= 64 bytes), outlen <= 128 bytes), thread per row (hybrid.cu shake_kernel); inlen and
// outlen multiples of 8, rows 4-byte aligned.
void shake256_rows(const uint8_t* in, size_t in_stride, int inlen, uint8_t* out, size_t out_stride, int outlen, size_t n,
                   cudaStream_t st);
// out[i] = KeyGen(k[i]) when p is null, else Shared(k[i], p[i]), for X25519 (hybrid.cu x25519_base_kernel /
// x25519_kernel) and X448 (x448_kernel), timed under KID_X25519 / KID_X448.  status[i] |= 1 where p[i] is of low order
// (status may be null).  Rows 4-byte aligned; a stride of 0 reads one row for the whole batch.
void x25519_rows(const uint8_t* k, size_t k_stride, const uint8_t* p, size_t p_stride, uint8_t* out, size_t out_stride,
                 uint8_t* status, size_t n, cudaStream_t st);
void x448_rows(const uint8_t* k, size_t k_stride, const uint8_t* p, size_t p_stride, uint8_t* out, size_t out_stride,
               uint8_t* status, size_t n, cudaStream_t st);
// The same for P-256 (p256.cu p256_base_kernel / p256_kernel, timed under KID_P256): scalars of 32 bytes, points and
// KeyGen outputs of 65 (0x04 || X || Y), Shared outputs of 32 (X), all big-endian and at any byte.  status[i] |= 1
// where p[i] is not a valid public key and |= 2 where k[i] is not a valid private key; that op's output is all zero.
void p256_rows(const uint8_t* k, size_t k_stride, const uint8_t* p, size_t p_stride, uint8_t* out, size_t out_stride,
               uint8_t* status, size_t n, cudaStream_t st);
// The same for P-384 (p384_base_kernel / p384_kernel, KID_P384: scalars and Shared outputs of 48 bytes, points and
// KeyGen outputs of 97) and P-521 (p521_*, KID_P521: 66 and 133 bytes).
void p384_rows(const uint8_t* k, size_t k_stride, const uint8_t* p, size_t p_stride, uint8_t* out, size_t out_stride,
               uint8_t* status, size_t n, cudaStream_t st);
void p521_rows(const uint8_t* k, size_t k_stride, const uint8_t* p, size_t p_stride, uint8_t* out, size_t out_stride,
               uint8_t* status, size_t n, cudaStream_t st);
}  // namespace hybrid
}  // namespace cb200
