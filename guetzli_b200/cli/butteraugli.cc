// Stand-alone `butteraugli` comparison tool on the device kernels (scope row f4):
//   butteraugli image1.png image2.png [heatmap.ppm]
// Interface, messages, score format and heat map of
// third_party/butteraugli/butteraugli/butteraugli_main.cc:362-455; the distance map
// comes from gb200_butteraugli_diffmap_srgb (the tool's sRGB conversion and alpha rule in front of
// ButteraugliInterface, butteraugli.cc:1858).
// A JPEG argument (FF D8, as the tool sniffs it, butteraugli_main.cc:282-307) is decoded on the device by
// gb200_jpeg_decode_rgb into the pixels the tool's ReadJPEG gets from libjpeg-turbo (RGB, gray replicated);
// a file that decoder refuses is reported as the tool reports a JPEG it cannot read.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "guetzli_b200.h"
#include "png_reader.h"

namespace {

struct Picture {
  int w = 0, h = 0;
  bool has_alpha = false;
  std::vector<uint8_t> rgba;
};

bool ReadAll(const char* name, std::string* out) {
  FILE* f = fopen(name, "rb");
  if (!f) {
    fprintf(stderr, "Cannot open %s\n", name);
    return false;
  }
  char buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}

Picture ReadImageOrDie(const char* name) {
  std::string data;
  if (!ReadAll(name, &data)) exit(1);
  if (data.size() < 2) {
    fprintf(stderr, "Cannot read from %s\n", name);
    exit(1);
  }
  Picture p;
  if (static_cast<uint8_t>(data[0]) == 0xff && static_cast<uint8_t>(data[1]) == 0xd8) {
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(data.data());
    const size_t len = data.size();
    std::vector<uint8_t> rgb;
    bool ok = gb200_jpeg_dimensions(bytes, len, &p.w, &p.h) != 0;
    if (ok) {
      rgb.resize(static_cast<size_t>(3) * p.w * p.h);
      uint8_t* out = rgb.data();
      int device = 0;
      if (const char* e = getenv("GUETZLI_B200_DEVICE")) device = atoi(e);
      ok = gb200_jpeg_decode_rgb(&bytes, &len, 1, device, &out) != 0;
    }
    if (!ok) {
      fprintf(stderr, "File %s is a malformed JPEG.\n", name);
      exit(1);
    }
    p.rgba.resize(static_cast<size_t>(4) * p.w * p.h);
    for (size_t i = 0; i < static_cast<size_t>(p.w) * p.h; ++i) {
      for (int c = 0; c < 3; ++c) p.rgba[4 * i + c] = rgb[3 * i + c];
      p.rgba[4 * i + 3] = 255;
    }
    return p;
  }
  if (!gb200_cli::ReadPNGRGBA(data, &p.w, &p.h, &p.rgba, &p.has_alpha)) {
    fprintf(stderr, "File %s is neither a valid JPEG nor a valid PNG.\n", name);
    exit(1);
  }
  return p;
}

// butteraugli.cc:1902 / :1923
double FuzzyClass(double score) {
  const double width_up = 6.07887388532, width_down = 5.50793514384, m0 = 2.0, scaler = 0.840253347958;
  if (score < 1.0) {
    double v = m0 / (1.0 + exp((score - 1.0) * width_down));
    v -= 1.0;
    v *= 2.0 - scaler;
    return v + scaler;
  }
  return m0 / (1.0 + exp((score - 1.0) * width_up)) * scaler;
}
double FuzzyInverse(double seek) {
  double pos = 0;
  for (double range = 1.0; range >= 1e-10; range *= 0.5) pos += FuzzyClass(pos) < seek ? -range : range;
  return pos;
}

// butteraugli_main.cc:311
void ScoreToRgb(double score, double good, double bad, uint8_t rgb[3]) {
  static const double kMap[12][3] = {{0, 0, 0}, {0, 0, 1}, {0, 1, 1}, {0, 1, 0},       {1, 1, 0},       {1, 0, 0},
                                     {1, 0, 1}, {0.5, 0.5, 1.0}, {1.0, 0.5, 0.5}, {1.0, 1.0, 0.5}, {1, 1, 1}, {1, 1, 1}};
  if (score < good) {
    score = (score / good) * 0.3;
  } else if (score < bad) {
    score = 0.3 + (score - good) / (bad - good) * 0.15;
  } else {
    score = 0.45 + (score - bad) / (bad * 12) * 0.5;
  }
  score = std::min<double>(std::max<double>(score * 11, 0.0), 10);
  const int ix = static_cast<int>(score);
  const double mix = score - ix;
  for (int i = 0; i < 3; ++i) {
    const double v = mix * kMap[ix + 1][i] + (1 - mix) * kMap[ix][i];
    rgb[i] = static_cast<uint8_t>(255 * pow(v, 0.5) + 0.5);
  }
}

// The tool's comparison (butteraugli_main.cc:239-281, :390-419): with alpha over black and over white,
// the larger distance and its map win.
bool Compare(const Picture& a, const Picture& b, int device, std::vector<float>* map, double* value) {
  const int channels = a.has_alpha ? 4 : 3;
  std::vector<uint8_t> rgb0, rgb1;
  const uint8_t* p0 = a.rgba.data();
  const uint8_t* p1 = b.rgba.data();
  if (channels == 3) {  // the reader gives RGBA
    const size_t n = static_cast<size_t>(a.w) * a.h;
    rgb0.resize(3 * n);
    rgb1.resize(3 * n);
    for (size_t i = 0; i < n; ++i)
      for (int c = 0; c < 3; ++c) {
        rgb0[3 * i + c] = a.rgba[4 * i + c];
        rgb1[3 * i + c] = b.rgba[4 * i + c];
      }
    p0 = rgb0.data();
    p1 = rgb1.data();
  }
  map->resize(static_cast<size_t>(a.w) * a.h);
  if (!gb200_butteraugli_diffmap_srgb(p0, p1, a.w, a.h, channels, device, map->data(), value)) {
    fprintf(stderr, "Butteraugli comparison failed\n");
    if (*gb200_last_error()) fprintf(stderr, "%s\n", gb200_last_error());
    return false;
  }
  return true;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 3 && argc != 4) {
    fprintf(stderr, "Usage: %s {image1.(png|jpg|jpeg)} {image2.(png|jpg|jpeg)} [heatmap.ppm]\n", argv[0]);
    return 1;
  }
  const Picture a = ReadImageOrDie(argv[1]);
  const Picture b = ReadImageOrDie(argv[2]);
  if (a.has_alpha != b.has_alpha) {
    fprintf(stderr, "Different number of channels: %lu vs %lu\n", a.has_alpha ? 4ul : 3ul, b.has_alpha ? 4ul : 3ul);
    return 1;
  }
  if (a.w != b.w || a.h != b.h) {
    fprintf(stderr, "The images are not equal in size: (%lu,%lu) vs (%lu,%lu)\n", static_cast<unsigned long>(a.w),
            static_cast<unsigned long>(b.w), static_cast<unsigned long>(a.h), static_cast<unsigned long>(b.h));
    return 1;
  }
  int device = 0;
  if (const char* e = getenv("GUETZLI_B200_DEVICE")) device = atoi(e);
  std::vector<float> map;
  double value = 0;
  if (!Compare(a, b, device, &map, &value)) return 1;
  printf("%lf\n", value);
  if (argc == 4) {
    const double good = FuzzyInverse(1.5), bad = FuzzyInverse(0.5);
    std::vector<uint8_t> rgb(3 * map.size());
    for (size_t i = 0; i < map.size(); ++i) ScoreToRgb(map[i], good, bad, &rgb[3 * i]);
    FILE* f = fopen(argv[3], "wb");
    if (f == NULL) {
      fprintf(stderr, "Cannot open %s\n", argv[3]);
      perror("fopen");
      return 1;
    }
    bool ok = fprintf(f, "P6\n%lu %lu\n255\n", static_cast<unsigned long>(a.w), static_cast<unsigned long>(a.h)) >= 0;
    ok = ok && fwrite(rgb.data(), 1, rgb.size(), f) == rgb.size();
    if (fclose(f) != 0) ok = false;
    if (!ok) return 1;
  }
  return 0;
}
