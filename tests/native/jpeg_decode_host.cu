// Host build of csrc/jpeg_decode.cuh for tests/test_jpeg_decode_cpu.py.  For each file it runs the decode twice: once
// sequentially (each restart interval from its start), and once as csrc/jpeg_decode.cu runs it: every subsequence from
// a guessed state, then synchronisation rounds until no entry changes, the block and DC scans, and the final pass, here
// taken over the subsequences in reverse order so that no pass can lean on its predecessor having run.
// Input records: [i32 h, w, luma_h, luma_v, subsequence bytes, interval count][i64 byte start, byte end, first MCU,
// MCUs per interval][i32 tables[kTableWords]][i64 scan length][scan bytes].
// Output records: [i32 sequential status, parallel status, rounds, agree][h * w * 3 bytes when the parallel status is
// 0]; the two agree when both statuses are nonzero or both are 0 with equal arrays (on a corrupt stream the parallel
// pass reports the largest status of its subsequences, not necessarily the first error).
#include <stdio.h>
#include <string.h>

#include <vector>

#include "jpeg_decode.cuh"

using namespace b200::jpeg_decode;

static bool read_all(void* p, size_t n) { return fread(p, 1, n, stdin) == n; }

struct Interval {
  long long a, b, m0, m;
};

// IDCT and colour conversion of decoded coefficients; returns the status.
static int finish(const Tables& t, const Geometry& g, const std::vector<int16_t>& coef, std::vector<uint8_t>& img) {
  std::vector<uint8_t> plane[3];
  for (int c = 0; c < 3; ++c) plane[c].assign(g.plane_bytes(c), 0);
  int st = kOk;
  for (long long b = 0; b < g.blocks; ++b) {
    int comp, bx, by;
    block_place(g, b, &comp, &bx, &by);
    const int pw = g.plane_w[comp];
    if (idct_islow(coef.data() + b * 64, t.quant[comp], plane[comp].data() + (long long)by * 8 * pw + bx * 8, pw))
      st = kRange;
  }
  img.assign((size_t)g.h * g.w * 3, 0);
  for (int y = 0; y < g.h; ++y)
    for (int x = 0; x < g.w; ++x)
      ycc_to_rgb(plane[0][(long long)y * g.plane_w[0] + x], chroma_at(g, plane[1].data(), g.plane_w[1], x, y),
                 chroma_at(g, plane[2].data(), g.plane_w[2], x, y), img.data() + ((size_t)y * g.w + x) * 3);
  return st;
}

static int sequential(const Tables& t, const Geometry& g, const uint8_t* scan, const std::vector<Interval>& ivs,
                      std::vector<uint8_t>& img) {
  std::vector<int16_t> coef(g.blocks * 64, 0);
  for (const Interval& iv : ivs) {
    const long long first = iv.m0 * g.bpm, blocks = iv.m * g.bpm;
    WriteSink sink{coef.data(), first, first + blocks, {0, 0, 0}};
    unsigned long long st = pack(iv.a * 8, 0, 0);
    const int s = run<true>(t, g, scan, iv.b * 8, iv.b * 8, blocks, &st, sink);
    if (s) return s;
    if (sink.at < first + blocks) return kShortStream;
    if (iv.b * 8 - pos_of(st) >= 8) return kTrailing;
  }
  return finish(t, g, coef, img);
}

static int parallel(const Tables& t, const Geometry& g, const uint8_t* scan, const std::vector<Interval>& ivs,
                    long long sub_bytes, int* rounds, std::vector<uint8_t>& img) {
  struct Sub {
    int iv;
    long long start, stop;
    bool first, last;
    long long iv_first;
  };
  std::vector<Sub> subs;
  for (int k = 0; k < (int)ivs.size(); ++k) {
    const long long first = subs.size();
    for (long long a = ivs[k].a; a < ivs[k].b; a += sub_bytes) {
      const long long b = a + sub_bytes < ivs[k].b ? a + sub_bytes : ivs[k].b;
      subs.push_back(Sub{k, a * 8, b * 8, a == ivs[k].a, b == ivs[k].b, first});
    }
  }
  const long long n = subs.size();
  std::vector<Exit> ex[2] = {std::vector<Exit>(n), std::vector<Exit>(n)};
  std::vector<unsigned long long> used(n);
  for (long long j = 0; j < n; ++j) {
    const Sub& s = subs[j];
    used[j] = pack(s.start, 0, 0);
    ex[0][j] = decode_sub(t, g, scan, ivs[s.iv].b * 8, s.stop, used[j]);
  }
  int cur = 0, r = 1;
  for (;; ++r) {
    bool changed = false;
    for (long long j = 0; j < n; ++j) {
      const Sub& s = subs[j];
      const unsigned long long entry = s.first ? pack(s.start, 0, 0) : ex[cur][j - 1].state;
      if (entry != used[j]) {
        changed = true;
        used[j] = entry;
        ex[cur ^ 1][j] = decode_sub(t, g, scan, ivs[s.iv].b * 8, s.stop, entry);
      } else {
        ex[cur ^ 1][j] = ex[cur][j];
      }
    }
    cur ^= 1;
    if (!changed) break;
  }
  *rounds = r - 1;
  std::vector<long long> prefix(4 * n);
  long long run_sum[4] = {0, 0, 0, 0};
  for (long long j = 0; j < n; ++j) {
    const Exit& e = ex[cur][j];
    for (int q = 0; q < 4; ++q) prefix[4 * j + q] = run_sum[q];
    run_sum[0] += e.count, run_sum[1] += e.dc[0], run_sum[2] += e.dc[1], run_sum[3] += e.dc[2];
  }
  std::vector<int16_t> coef(g.blocks * 64, 0);
  int status = kOk;
  for (long long j = n - 1; j >= 0; --j) {
    const Sub& s = subs[j];
    const Interval& iv = ivs[s.iv];
    const long long first = iv.m0 * g.bpm, blocks = iv.m * g.bpm, end = iv.b * 8;
    const unsigned long long entry = s.first ? pack(s.start, 0, 0) : ex[cur][j - 1].state;
    const long long* p = &prefix[4 * j];
    const long long* p0 = &prefix[4 * s.iv_first];
    const long long rel = p[0] - p0[0];
    WriteSink sink{coef.data(), first + rel, first + blocks,
                   {(int)(p[1] - p0[1]), (int)(p[2] - p0[2]), (int)(p[3] - p0[3])}};
    int st = kOk;
    if (entry == kInvalid) continue;
    if (s.last && (rel > blocks || (rel == blocks && zz_of(entry) != 0))) {
      st = kTrailing;
    } else {
      unsigned long long e = entry;
      st = run<true>(t, g, scan, end, s.stop, s.last ? blocks - rel : (long long)1 << 62, &e, sink);
      if (st == kOk && sink.overflow) st = kTrailing;
      if (st == kOk && s.last) {
        if (sink.at < first + blocks || pos_of(e) > end) st = kShortStream;
        else if (end - pos_of(e) >= 8) st = kTrailing;
      }
    }
    if (st > status) status = st;
  }
  if (status) return status;
  return finish(t, g, coef, img);
}

int main() {
  for (;;) {
    int32_t head[6];
    if (!read_all(head, sizeof(head))) break;
    std::vector<Interval> ivs(head[5]);
    if (head[5] && !read_all(ivs.data(), sizeof(Interval) * ivs.size())) return 1;
    Tables* t = new Tables;
    long long len;
    if (!read_all(t, sizeof(Tables)) || !read_all(&len, 8)) return 1;
    std::vector<uint8_t> scan(len ? len : 1);
    if (!read_all(scan.data(), len)) return 1;
    Geometry g;
    if (!geometry_of(head[0], head[1], head[2], head[3], &g)) return 2;
    std::vector<uint8_t> a, b;
    int rounds = 0;
    const int32_t s1 = sequential(*t, g, scan.data(), ivs, a);
    const int32_t s2 = parallel(*t, g, scan.data(), ivs, head[4], &rounds, b);
    const int32_t out[4] = {s1, s2, rounds, (int32_t)((s1 == 0) == (s2 == 0) && (s1 != 0 || a == b))};
    fwrite(out, 4, 4, stdout);
    if (s2 == kOk) fwrite(b.data(), 1, b.size(), stdout);
    delete t;
  }
  return 0;
}
