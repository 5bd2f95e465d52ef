// Evidence for the heat-map kernel's output byte (HeatMap, kernels.h), ScoreToRgb's
// (uint8_t)(255 * pow(v, 0.5) + 0.5) (b/butteraugli.cc:1973), on this host's libm:
//   - the kernel looks the byte up in a table of steps, built by bisection with this pow as heat_byte_steps()
//     (tables.cc) builds it: [k] = the least double v in [0, 1] whose byte is at least k.  On a window of 2^W ulps
//     either side of every step the table's byte is compared with pow's byte (pow is at most an ulp from the
//     correctly rounded sqrt, so outside these windows neither byte can change);
//   - IEEE sqrt(v) in place of pow(v, 0.5) is compared on the same windows, as doubles and as bytes.
// Prints every byte difference; exits 1 if the table differs from pow anywhere.
//   g++ -O2 -ffp-contract=off -o /tmp/heatmap_byte_check tools/heatmap_byte_check.cc && /tmp/heatmap_byte_check 16
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static double of_bits(uint64_t b) {
  double v;
  memcpy(&v, &b, 8);
  return v;
}
static uint64_t bits_of(double v) {
  uint64_t b;
  memcpy(&b, &v, 8);
  return b;
}
static int byte_of(double r) { return static_cast<uint8_t>(255 * r + 0.5); }

int main(int argc, char** argv) {
  const int W = argc > 1 ? atoi(argv[1]) : 16;
  double steps[256] = {0};
  for (int k = 1; k <= 255; ++k) {
    uint64_t lo = 0, hi = bits_of(1.0);
    while (hi - lo > 1) {
      const uint64_t mid = lo + (hi - lo) / 2;
      (byte_of(pow(of_bits(mid), 0.5)) >= k ? hi : lo) = mid;
    }
    steps[k] = of_bits(hi);
  }
  long long checked = 0, table_diffs = 0, sqrt_value_diffs = 0, sqrt_byte_diffs = 0;
  for (int k = 1; k <= 255; ++k) {
    for (long long d = -(1LL << W); d <= (1LL << W); ++d) {
      const double v = of_bits(bits_of(steps[k]) + d);
      if (!(v >= 0 && v <= 1)) continue;
      const double p = pow(v, 0.5), s = sqrt(v);
      int t = 0;
      for (int step = 128; step > 0; step >>= 1)
        if (t + step <= 255 && steps[t + step] <= v) t += step;
      ++checked;
      if (t != byte_of(p)) {
        ++table_diffs;
        printf("table: k=%d v=%.17g pow byte %d, table byte %d\n", k, v, byte_of(p), t);
      }
      if (p != s) ++sqrt_value_diffs;
      if (byte_of(p) != byte_of(s)) {
        ++sqrt_byte_diffs;
        printf("sqrt: k=%d v=%.17g (bits %016llx) pow=%.17g byte %d, sqrt=%.17g byte %d\n", k, v,
               static_cast<unsigned long long>(bits_of(v)), p, byte_of(p), s, byte_of(s));
      }
    }
  }
  printf("%lld values around 255 steps (2^%d ulps either side): table %lld byte differences; sqrt %lld value and "
         "%lld byte differences\n", checked, W, table_diffs, sqrt_value_diffs, sqrt_byte_diffs);
  return table_diffs ? 1 : 0;
}
