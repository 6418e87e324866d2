// Baseline JPEG decoded on the device, array for array what Pillow (libjpeg-turbo) gives (deva/utils/jpeg_decode.py;
// the format rules are DESIGN §7).  The host has parsed each file, checked its markers, removed the stuffing bytes and
// RSTn markers from the scan and cut every restart interval into subsequences of a fixed number of bytes.  Then:
//   1. zero_kernel clears the files' coefficient blocks.
//   2. sync_kernel, one cooperative launch: every subsequence is decoded from a guessed state (its first bit, slot 0,
//      zig-zag index 0) to the state at which it leaves (jpeg_decode.cuh).  Then, round by round, every subsequence
//      whose predecessor's exit state differs from the entry it was decoded from is decoded again from that exit,
//      until one round changes no entry; the first subsequence of a restart interval starts in its known state.  A
//      fixed point is the sequential decode, and the rounds are decided on the device, between grid barriers.  The
//      same launch then scans the subsequences' block counts and per-component DC sums.
//   3. write_kernel decodes every subsequence once more from its true entry and writes int16 coefficients in block
//      order, the DC values running from the predictors the scan gave (reset at each restart interval); the last
//      subsequence of an interval checks that exactly the interval's blocks were decoded and at most 7 padding bits
//      remain.
//   4. idct_kernel: one thread per block, jidctint.c's islow IDCT into per-component sample planes.
//   5. color_kernel: one thread per pixel, fancy upsampling and YCbCr -> RGB into [h, w, 3].
// Every read of the scan is bounded by the interval's end and every write by the file's shape; a malformed file gets
// a nonzero status and no fault.
#include <algorithm>
#include <cooperative_groups.h>
#include <stdint.h>

#include "common.h"
#include "jpeg_decode.cuh"
#include "scan.cuh"

namespace b200 {
namespace jpeg_decode {

namespace cg = cooperative_groups;

constexpr int kSyncThreads = 256;
constexpr int kMaxSyncBlocks = 1024;
constexpr int kThreads = 256;

// The batch's shared part of the workspace.
struct Shared {
  int flags[3];   // round r sets flags[r % 3] when an entry changed
  int rounds;     // rounds the last batch took (0 = the guesses were right everywhere)
  int final_buf;  // which exit buffer holds the fixed point
  int pad[3];
  long long block_sums[kMaxSyncBlocks][4];
};

// One file's part: its coefficients, sample planes and the state of its subsequences.
struct FileWork {
  int16_t* coef;
  uint8_t* plane[3];
  Exit* exits[2];
  unsigned long long* used;
  long long (*prefix)[4];
};

template <class C>
__host__ __device__ inline FileWork carve(C& c, const Geometry& g, long long subs) {
  FileWork w;
  w.coef = c.template take<int16_t>(g.blocks * 64);
  for (int k = 0; k < 3; ++k) w.plane[k] = c.template take<uint8_t>(g.plane_bytes(k));
  w.exits[0] = c.template take<Exit>(subs);
  w.exits[1] = c.template take<Exit>(subs);
  w.used = c.template take<unsigned long long>(subs);
  w.prefix = reinterpret_cast<long long(*)[4]>(c.template take<long long>(subs * 4));
  return w;
}

struct Args {
  const uint8_t* scans;
  const int64_t* desc;
  int n;
  const int32_t* tables;
  const int64_t* intervals;
  long long n_iv;
  const int64_t* subs;
  long long n_sub;
  uint8_t* out;
  Shared* shared;
  char* files;
  int32_t* status;
};

__device__ inline bool file_view(const Args& a, int f, Geometry* g, FileWork* w) {
  const int64_t* d = a.desc + (size_t)f * kDescFields;
  if (!geometry_of(d[kH], d[kW], d[kLumaH], d[kLumaV], g) || d[kScanOff] < 0 || d[kScanLen] < 0 || d[kOutOff] < 0 ||
      d[kWorkOff] < 0 || d[kTablesIdx] < 0 || d[kTablesIdx] >= a.n || d[kFirstSub] < 0 || d[kSubs] < 1 ||
      d[kFirstSub] + d[kSubs] > a.n_sub)
    return false;
  Carver<16> c{a.files + d[kWorkOff]};
  *w = carve(c, *g, d[kSubs]);
  return true;
}

// Everything a thread needs about subsequence j; ok is false when its records are out of range.
struct SubView {
  bool ok = false;
  int f;
  Geometry g;
  FileWork w;
  const Tables* t;
  long long local, iv_local, start, stop, end, iv_start, first_block, blocks;
  bool first, last;
};

__device__ inline SubView sub_view(const Args& a, long long j) {
  SubView v;
  const int64_t* s = a.subs + j * kSubFields;
  if (s[kSubInterval] < 0 || s[kSubInterval] >= a.n_iv) return v;
  const int64_t* iv = a.intervals + s[kSubInterval] * kIvFields;
  if (iv[kIvFile] < 0 || iv[kIvFile] >= a.n) return v;
  v.f = (int)iv[kIvFile];
  if (!file_view(a, v.f, &v.g, &v.w)) return v;
  const int64_t* d = a.desc + (size_t)v.f * kDescFields;
  const long long lo = d[kScanOff] * 8, hi = (d[kScanOff] + d[kScanLen]) * 8;
  v.start = s[kSubBitStart], v.stop = s[kSubBitEnd], v.iv_start = iv[kIvBitStart], v.end = iv[kIvBitEnd];
  v.first_block = iv[kIvFirstBlock], v.blocks = iv[kIvBlocks];
  if (v.iv_start < lo || v.end > hi || v.iv_start > v.end || v.start < v.iv_start || v.stop > v.end ||
      v.start >= v.stop || v.first_block < 0 || v.blocks < 0 || v.first_block + v.blocks > v.g.blocks ||
      iv[kIvFirstSub] < d[kFirstSub] || iv[kIvFirstSub] > j || j >= d[kFirstSub] + d[kSubs] || (v.iv_start & 7) ||
      (v.end & 7))
    return v;
  v.local = j - d[kFirstSub];
  v.iv_local = iv[kIvFirstSub] - d[kFirstSub];
  v.first = j == iv[kIvFirstSub];
  v.last = v.stop == v.end;
  v.t = reinterpret_cast<const Tables*>(a.tables) + d[kTablesIdx];
  v.ok = true;
  return v;
}

__device__ inline void fail(int32_t* status, int f, int st) {
  if (st != kOk) atomicMax(status + f, st);
}

__global__ void __launch_bounds__(kThreads) zero_kernel(Args a) {
  const int f = blockIdx.y;
  Geometry g;
  FileWork w;
  if (!file_view(a, f, &g, &w)) {
    if (threadIdx.x == 0 && blockIdx.x == 0) fail(a.status, f, kBadDescriptor);
    return;
  }
  uint4* p = reinterpret_cast<uint4*>(w.coef);
  const long long n = g.blocks * 8;  // 128 bytes per block
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    p[i] = make_uint4(0, 0, 0, 0);
}

__global__ void __launch_bounds__(kSyncThreads) sync_kernel(Args a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ long long warp_sums[kSyncThreads / 32];
  const long long threads = (long long)gridDim.x * blockDim.x;
  const long long per = (a.n_sub + threads - 1) / threads;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long j0 = min(a.n_sub, t * per), j1 = min(a.n_sub, j0 + per);
  Shared& sh = *a.shared;

  for (long long j = j0; j < j1; ++j) {
    SubView v = sub_view(a, j);
    if (!v.ok) continue;
    const unsigned long long entry = pack(v.first ? v.iv_start : v.start, 0, 0);
    v.w.used[v.local] = entry;
    v.w.exits[0][v.local] = decode_sub(*v.t, v.g, a.scans, v.end, v.stop, entry);
  }
  grid.sync();
  int cur = 0, r = 1;
  for (;; ++r) {
    bool changed = false;
    for (long long j = j0; j < j1; ++j) {
      SubView v = sub_view(a, j);
      if (!v.ok) continue;
      const Exit* in = v.w.exits[cur];
      Exit* nx = v.w.exits[cur ^ 1];
      const unsigned long long entry = v.first ? pack(v.iv_start, 0, 0) : in[v.local - 1].state;
      if (entry != v.w.used[v.local]) {
        changed = true;
        v.w.used[v.local] = entry;
        nx[v.local] = decode_sub(*v.t, v.g, a.scans, v.end, v.stop, entry);
      } else {
        nx[v.local] = in[v.local];
      }
    }
    if (t == 0) sh.flags[(r + 1) % 3] = 0;
    if (changed) sh.flags[r % 3] = 1;
    grid.sync();
    cur ^= 1;
    if (!*(volatile int*)&sh.flags[r % 3]) break;
  }
  if (t == 0) sh.rounds = r - 1, sh.final_buf = cur;

  // Exclusive prefix sums over all subsequences of (blocks, DC sum per component).
  long long mine[4] = {0, 0, 0, 0};
  for (long long j = j0; j < j1; ++j) {
    SubView v = sub_view(a, j);
    if (!v.ok) continue;
    const Exit& e = v.w.exits[cur][v.local];
    mine[0] += e.count, mine[1] += e.dc[0], mine[2] += e.dc[1], mine[3] += e.dc[2];
  }
  long long before[4];
  for (int q = 0; q < 4; ++q) {
    long long total;
    before[q] = block_exclusive_scan(mine[q], warp_sums, total);
    if (threadIdx.x == 0) sh.block_sums[blockIdx.x][q] = total;
  }
  grid.sync();
  for (int q = 0; q < 4; ++q)
    for (int b = 0; b < (int)blockIdx.x; ++b) before[q] += sh.block_sums[b][q];
  for (long long j = j0; j < j1; ++j) {
    SubView v = sub_view(a, j);
    if (!v.ok) continue;
    const Exit& e = v.w.exits[cur][v.local];
    for (int q = 0; q < 4; ++q) v.w.prefix[v.local][q] = before[q];
    before[0] += e.count, before[1] += e.dc[0], before[2] += e.dc[1], before[3] += e.dc[2];
  }
}

__global__ void __launch_bounds__(kThreads) write_kernel(Args a) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n_sub) return;
  const SubView v = sub_view(a, j);
  if (!v.ok) {
    const int64_t iv = a.subs[j * kSubFields + kSubInterval];
    if (iv >= 0 && iv < a.n_iv) {
      const int64_t f = a.intervals[iv * kIvFields + kIvFile];
      if (f >= 0 && f < a.n) fail(a.status, (int)f, kBadDescriptor);
    }
    return;
  }
  const Exit* ex = v.w.exits[a.shared->final_buf];
  const unsigned long long entry = v.first ? pack(v.iv_start, 0, 0) : ex[v.local - 1].state;
  const long long* p = v.w.prefix[v.local];
  const long long* p0 = v.w.prefix[v.iv_local];
  const long long rel = p[0] - p0[0];
  WriteSink sink{v.w.coef, v.first_block + rel, v.first_block + v.blocks,
                 {(int)(p[1] - p0[1]), (int)(p[2] - p0[2]), (int)(p[3] - p0[3])}};
  if (entry == kInvalid) return;  // the subsequence that failed reports it
  if (v.last && (rel > v.blocks || (rel == v.blocks && zz_of(entry) != 0))) return fail(a.status, v.f, kTrailing);
  unsigned long long st = entry;
  const int s = run<true>(*v.t, v.g, a.scans, v.end, v.stop, v.last ? v.blocks - rel : (long long)1 << 62, &st, sink);
  if (s != kOk) return fail(a.status, v.f, s);
  if (sink.overflow) return fail(a.status, v.f, kTrailing);
  if (v.last) {
    const long long pos = pos_of(st);
    if (sink.at < v.first_block + v.blocks || pos > v.end) return fail(a.status, v.f, kShortStream);
    if (v.end - pos >= 8) return fail(a.status, v.f, kTrailing);
  }
}

__global__ void __launch_bounds__(kThreads) idct_kernel(Args a) {
  const int f = blockIdx.y;
  if (a.status[f] != kOk) return;
  Geometry g;
  FileWork w;
  if (!file_view(a, f, &g, &w)) return;
  const int32_t* quant = (reinterpret_cast<const Tables*>(a.tables) + a.desc[(size_t)f * kDescFields + kTablesIdx])
                             ->quant[0];
  int bad = kOk;
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < g.blocks;
       b += (long long)gridDim.x * blockDim.x) {
    int comp, bx, by;
    block_place(g, b, &comp, &bx, &by);
    const int pw = g.plane_w[comp];
    if (idct_islow(w.coef + b * 64, quant + comp * 64, w.plane[comp] + (long long)by * 8 * pw + bx * 8, pw) != kOk)
      bad = kRange;
  }
  if (bad != kOk) fail(a.status, f, bad);
}

__global__ void __launch_bounds__(kThreads) color_kernel(Args a) {
  const int f = blockIdx.y;
  if (a.status[f] != kOk) return;
  Geometry g;
  FileWork w;
  if (!file_view(a, f, &g, &w)) return;
  uint8_t* out = a.out + a.desc[(size_t)f * kDescFields + kOutOff];
  const long long n = (long long)g.h * g.w;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / g.w), x = (int)(i - (long long)y * g.w);
    const int yy = w.plane[0][(long long)y * g.plane_w[0] + x];
    const int cb = chroma_at(g, w.plane[1], g.plane_w[1], x, y);
    const int cr = chroma_at(g, w.plane[2], g.plane_w[2], x, y);
    ycc_to_rgb(yy, cb, cr, out + i * 3);
  }
}

}  // namespace jpeg_decode
}  // namespace b200

using namespace b200;

namespace {

size_t shared_bytes() { return (sizeof(jpeg_decode::Shared) + 15) / 16 * 16; }

// Cooperative blocks of sync_kernel that fit on the current device at once.
int sync_capacity() {
  static int cached[64];
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && cached[dev]) return cached[dev];
  int sms = 0, per_sm = 0;
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpeg_decode::sync_kernel,
                                                          jpeg_decode::kSyncThreads, 0));
  const int cap = std::min(jpeg_decode::kMaxSyncBlocks, sms * per_sm);
  if (dev < 64) cached[dev] = cap;
  return cap;
}

}  // namespace

extern "C" {

DEVA_B200_API size_t deva_b200_jpeg_decode_workspace_bytes(int h, int w, int luma_h, int luma_v,
                                                           int64_t subsequences) {
  if (h == 0 && w == 0) return shared_bytes();
  jpeg_decode::Geometry g;
  if (!jpeg_decode::geometry_of(h, w, luma_h, luma_v, &g) || subsequences < 0) return 0;
  Carver<16> c{nullptr};
  jpeg_decode::carve(c, g, subsequences);
  return c.bytes;
}

DEVA_B200_API int deva_b200_jpeg_decode(const uint8_t* scans, const int64_t* desc, int n, const int32_t* tables,
                                        const int64_t* intervals, int64_t n_intervals, const int64_t* subs,
                                        int64_t n_subs, uint8_t* out, void* workspace, int32_t* status,
                                        deva_stream_t stream) {
  B200_REQUIRE(n >= 0 && n_intervals >= 0 && n_subs >= 0 &&
                   (n == 0 || (scans && desc && tables && out && workspace && status)) &&
                   (n_subs == 0 || (intervals && subs)),
               "jpeg_decode: bad arguments");
  if (n == 0) return 0;
  cudaStream_t s = S(stream);
  jpeg_decode::Args a{scans,  desc, n, tables, intervals, n_intervals, subs, n_subs, out,
                      static_cast<jpeg_decode::Shared*>(workspace),
                      static_cast<char*>(workspace) + shared_bytes(), status};
  B200_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * n, s));
  B200_CUDA(cudaMemsetAsync(workspace, 0, sizeof(jpeg_decode::Shared), s));
  B200_REQUIRE(n <= 65535, "jpeg_decode: at most 65535 files per batch");
  const dim3 per_file(64, n);
  jpeg_decode::zero_kernel<<<per_file, jpeg_decode::kThreads, 0, s>>>(a);
  B200_LAUNCH_CHECK();
  if (n_subs > 0) {
    const long long want = (n_subs + jpeg_decode::kSyncThreads - 1) / jpeg_decode::kSyncThreads;
    const int blocks = (int)std::min<long long>(want, sync_capacity());
    void* args[] = {&a};
    B200_CUDA(cudaLaunchCooperativeKernel((const void*)jpeg_decode::sync_kernel, dim3(blocks),
                                          dim3(jpeg_decode::kSyncThreads), args, 0, s));
    B200_LAUNCH_CHECK();
    jpeg_decode::write_kernel<<<(unsigned)((n_subs + jpeg_decode::kThreads - 1) / jpeg_decode::kThreads),
                                jpeg_decode::kThreads, 0, s>>>(a);
    B200_LAUNCH_CHECK();
  }
  jpeg_decode::idct_kernel<<<per_file, jpeg_decode::kThreads, 0, s>>>(a);
  B200_LAUNCH_CHECK();
  jpeg_decode::color_kernel<<<dim3(256, n), jpeg_decode::kThreads, 0, s>>>(a);
  B200_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
