// JPEG input (row f2 of the scope table): parses a baseline / extended-sequential /
// progressive Huffman JPEG into quantised DCT coefficients, the way the reference's
// ReadJpeg(JPEG_READ_ALL) does (g/jpeg_data_reader.cc:931): same accepted streams,
// same coefficient values, quant tables, APPn / COM payloads and tail bytes.  Host
// code; the coefficients then go to the device exactly like freshly encoded ones.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

namespace gb200 {

struct JpegQuantTable {
  int values[64];  // natural (row-major) order
  int precision;   // 0: 8 bit, 1: 16 bit entries in the DQT segment
  int index;       // Tq
};

struct JpegComponent {
  int id;
  int h_samp, v_samp;
  int quant_idx;  // index into JpegInput::quant (after the Tq fix-up)
  int width_in_blocks, height_in_blocks;
  std::vector<int16_t> coeffs;  // [block][64], natural order, quantised
};

struct JpegInput {
  int width = 0, height = 0;
  int max_h = 1, max_v = 1;
  int mcu_cols = 0, mcu_rows = 0;
  std::vector<JpegComponent> components;
  std::vector<JpegQuantTable> quant;
  std::vector<std::string> app_data;  // marker low byte + length bytes + payload (g/jpeg_data_reader.cc:396)
  std::vector<std::string> com_data;  // length bytes + payload (:411)
  std::string tail_data;              // bytes after EOI
  bool progressive = false;           // SOF2
  // per component and zig-zag position: bit b is set once a scan has coded bit b of that coefficient
  uint16_t coded_bits[4][64] = {};
  bool is_444() const;                // g/jpeg_data.cc:36
  bool is_420() const;                // g/jpeg_data.cc:24
};

// Canonical Huffman code of one DHT table, decoded by code length (decode_symbol in jpeg_in.cc).
struct JpegHuffTable {
  bool defined = false;
  int max_code[18];    // largest code of each length, -1 if none
  int val_offset[18];  // index of the first symbol of each length minus its first code
  uint8_t symbols[256];
  int num_symbols = 0;
};

// One SOS header: the frame's components it carries and their tables, spectral selection, approximation.
struct JpegScanSpec {
  int ncomp;
  int comp[4], dc_tbl[4], ac_tbl[4];
  int ss, se, ah, al;
};

// A file read up to and including its first SOS header (read_jpeg_header).
struct JpegScanHeader {
  JpegInput jpg;  // frame, quant tables (Tq fixed up as read_jpeg does), APPn / COM; no coefficients
  JpegHuffTable dc[4], ac[4];
  JpegScanSpec scan;
  int restart_interval = 0;
  size_t scan_start = 0;  // offset of the first byte of entropy-coded data
};

// Returns false (message in *err) for streams the reference rejects.
bool read_jpeg(const uint8_t* data, size_t len, JpegInput* jpg, std::string* err);

// read_jpeg up to the end of the first SOS header, with the same checks on what it reads and the ones
// read_jpeg makes after the last segment (quant tables found, DHT count); it prints nothing.  False if
// read_jpeg would refuse what was read, or if the bytes end first (data may be a prefix of the file).
bool read_jpeg_header(const uint8_t* data, size_t len, JpegScanHeader* hdr);

// ReadJpeg(JPEG_READ_HEADER): only the frame size (the CLI's memory-limit check,
// g/guetzli.cc:306-312).
bool read_jpeg_dimensions(const uint8_t* data, size_t len, int* width, int* height);

// g/jpeg_data_decoder.cc:24: libjpeg's colour space guess for three components.
bool has_ycbcr_color_space(const JpegInput& jpg);
// libjpeg-turbo's colour space guess for three components (default_decompress_parms, jdapimin.c): a
// JFIF APP0 (payload "JFIF\0" and at least 14 bytes) means YCbCr; else an Adobe APP14 (payload "Adobe",
// at least 12 bytes; the last one counts) means RGB for transform 0 and YCbCr otherwise; else component
// ids 'R', 'G', 'B' mean RGB and anything else YCbCr.  has_ycbcr_color_space is the guetzli reference's
// version of that guess, which does not look at the payloads (any APP0 means YCbCr, any APP14 of 15
// bytes or more is taken for Adobe's); the encoder keeps it.
bool libjpeg_ycbcr(const JpegInput& jpg);
// Whether libjpeg-turbo's jpeg_start_decompress, with the defaults the butteraugli tool's ReadJPEG leaves
// alone (b/butteraugli_main.cc:157-232), gives the pixels jpeg_decode_rgb (pipeline.h) computes from this
// parsed file; if not, the reason in *why.  Accepted: 1 component (gray), or 3 components whose first
// has the frame's maximum sampling of 1x1, 2x1 or 2x2 and whose other two are 1x1 (4:4:4, 4:2:2, 4:2:0);
// progressive files only where libjpeg does not block-smooth (smoothing_ok, jdcoefct.c); and only files
// whose blocks stay in the range where libjpeg-turbo's SIMD IDCT computes its C IDCT's samples (jpeg_islow).
bool libjpeg_decodable(const JpegInput& jpg, std::string* why);
// g/processor.cc:106: |coeff * quant| <= 4096 everywhere.
bool check_jpeg_sanity(const JpegInput& jpg);

}  // namespace gb200
