// Host build of csrc/inflate.cuh for tests/test_png_decode_cpu.py.  Reads records from stdin, each
// [u32 stream length][stream bytes][u64 expected inflated length], and writes for each
// [i32 status][u64 inflated length][the inflated bytes when the status is 0].  The output buffer is exactly the
// expected length, so any write past it would be a bug of the core, not of this driver.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "inflate.cuh"

using namespace b200::inflate;

static bool read_all(void* p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main() {
  Tables* t = new Tables;
  std::vector<uint8_t> win(kWindow);
  for (;;) {
    uint32_t len;
    if (!read_all(&len, 4)) break;
    std::vector<uint8_t> in(len ? len : 1);
    uint64_t out_len;
    if (!read_all(in.data(), len) || !read_all(&out_len, 8)) return 1;
    std::vector<uint8_t> out(out_len ? out_len : 1);
    Inflater s;
    s.init(in.data(), len, out.data(), (long long)out_len, win.data());
    int st;
    while ((st = s.run(*t, 16)) == kCopyPending)
      for (int j = 0; j < s.copy_len; ++j) s.put(s.copy_at + j, s.source(s.copy_at, s.copy_dist, j));
    if (st == kOk && adler32(out.data(), (long long)out_len) != s.adler) st = kBadAdler;
    const int32_t status = st;
    fwrite(&status, 4, 1, stdout);
    fwrite(&out_len, 8, 1, stdout);
    if (st == kOk) fwrite(out.data(), 1, out_len, stdout);
  }
  delete t;
  return 0;
}
