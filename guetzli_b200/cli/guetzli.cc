// `guetzli` command line on top of libguetzli_b200.so.
//
// Behavioural contract = the reference tool (guetzli/guetzli.cc:155-326, exercised by
// tests/smoke_test.sh): `guetzli [--verbose] [--quality Q] [--memlimit M] [--nomemlimit]
// [--] in out`, "-" for stdin / stdout, PNG or JPEG input told apart by the PNG signature,
// every failure (usage included) exits with 1 after the reference's message on stderr.
// The encoding itself is guetzli::Process of include/guetzli_b200_compat.h.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <exception>
#include <string>
#include <vector>

#include "guetzli_b200_compat.h"
#include "png_reader.h"

namespace {

struct Options {
  bool verbose = false;
  int quality = 95;        // --quality
  int memlimit_mb = 6000;  // --memlimit; -1 = --nomemlimit
  const char* input = nullptr;
  const char* output = nullptr;
};

[[noreturn]] void UsageAndExit() {
  static const char kText[] =
      "Guetzli JPEG compressor. Usage: \n"
      "guetzli [flags] input_filename output_filename\n"
      "\n"
      "Flags:\n"
      "  --verbose    - Print a verbose trace of all attempts to standard output.\n"
      "  --quality Q  - Visual quality to aim for, expressed as a JPEG quality value.\n"
      "                 Default value is %d.\n"
      "  --memlimit M - Memory limit in MB. Guetzli will fail if unable to stay under\n"
      "                 the limit. Default limit is %d MB.\n"
      "  --nomemlimit - Do not limit memory usage.\n"
      "\n"
      "This build (guetzli_b200) encodes YUV444 only: JPEG input with 4:2:0 chroma\n"
      "subsampling is refused (\"YUV420 JPEG input is outside the GPU hot path\");\n"
      "convert such files to PNG first.\n";
  const Options defaults;
  fprintf(stderr, kText, defaults.quality, defaults.memlimit_mb);
  exit(1);
}

[[noreturn]] void DieWithErrno(const char* what) {
  perror(what);
  exit(1);
}

// Flags are the leading arguments that start with "--"; a bare "--" ends them.  Exactly two
// positional arguments must remain.
Options ParseCommandLine(int argc, char** argv) {
  Options o;
  int i = 1;
  auto value_of = [&](int* into) {
    if (++i >= argc) UsageAndExit();
    *into = atoi(argv[i]);
  };
  while (i < argc && strncmp(argv[i], "--", 2) == 0) {
    const std::string flag = argv[i];
    if (flag == "--") {
      ++i;
      break;
    }
    if (flag == "--verbose") {
      o.verbose = true;
    } else if (flag == "--quality") {
      value_of(&o.quality);
    } else if (flag == "--memlimit") {
      value_of(&o.memlimit_mb);
    } else if (flag == "--nomemlimit") {
      o.memlimit_mb = -1;
    } else {
      fprintf(stderr, "Unknown commandline flag: %s\n", argv[i]);
      UsageAndExit();
    }
    ++i;
  }
  if (argc - i != 2) UsageAndExit();
  o.input = argv[i];
  o.output = argv[i + 1];
  return o;
}

bool IsDash(const char* name) { return name[0] == '-' && name[1] == '\0'; }

std::string Slurp(const char* name) {
  FILE* f = IsDash(name) ? stdin : fopen(name, "rb");
  if (f == nullptr) DieWithErrno("Can't open input file");
  std::string bytes;
  std::vector<char> chunk(1 << 16);
  size_t got;
  while ((got = fread(chunk.data(), 1, chunk.size(), f)) > 0) bytes.append(chunk.data(), got);
  if (ferror(f)) DieWithErrno("fread");
  if (f != stdin) fclose(f);
  return bytes;
}

void Spill(const char* name, const std::string& bytes) {
  FILE* f = IsDash(name) ? stdout : fopen(name, "wb");
  if (f == nullptr) DieWithErrno("Can't open output file for writing");
  if (fwrite(bytes.data(), 1, bytes.size(), f) != bytes.size()) DieWithErrno("fwrite");
  if (fclose(f) < 0) DieWithErrno("fclose");
}

// The reference budgets 350 bytes per pixel and refuses limits under 100 MB.
bool WithinMemoryLimit(const Options& o, int width, int height) {
  if (o.memlimit_mb == -1) return true;
  const double need_mb = static_cast<double>(width) * height * 350 / (1 << 20);
  return need_mb <= o.memlimit_mb && o.memlimit_mb >= 100;
}

bool LooksLikePng(const std::string& bytes) {
  static const unsigned char kSignature[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  return bytes.size() >= sizeof(kSignature) && memcmp(bytes.data(), kSignature, sizeof(kSignature)) == 0;
}

int Fail(const char* message) {
  fprintf(stderr, "%s\n", message);
  return 1;
}

void OnUnhandledException() {
  fprintf(stderr,
          "Unhandled exception. Most likely insufficient memory available.\n"
          "Make sure that there is 300MB/MPix of memory available.\n");
  exit(1);
}

}  // namespace

int main(int argc, char** argv) {
  std::set_terminate(OnUnhandledException);
  const Options opt = ParseCommandLine(argc, argv);
  const std::string input = Slurp(opt.input);

  guetzli::Params params;
  params.butteraugli_target = static_cast<float>(guetzli::ButteraugliScoreForQuality(opt.quality));
  guetzli::ProcessStats stats;
  if (opt.verbose) stats.debug_output_file = stderr;

  std::string jpeg;
  int width = 0, height = 0;
  bool ok;
  if (LooksLikePng(input)) {
    std::vector<uint8_t> rgb;
    if (!gb200_cli::ReadPNG(input, &width, &height, &rgb)) return Fail("Error reading PNG data from input file");
    if (!WithinMemoryLimit(opt, width, height)) return Fail("Memory limit would be exceeded. Failing.");
    ok = guetzli::Process(params, &stats, rgb, width, height, &jpeg);
  } else {
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(input.data());
    if (!gb200_jpeg_dimensions(bytes, input.size(), &width, &height))
      return Fail("Error reading JPG data from input file");
    if (!WithinMemoryLimit(opt, width, height)) return Fail("Memory limit would be exceeded. Failing.");
    ok = guetzli::Process(params, &stats, input, &jpeg);
  }
  if (!ok) return Fail("Guetzli processing failed");
  Spill(opt.output, jpeg);
  return 0;
}
