// JPEG input parser (ITU-T T.81 Huffman modes: SOF0 / SOF1 sequential, SOF2
// progressive with spectral selection and successive approximation, restart
// intervals).  Behavioural model: ReadJpeg(JPEG_READ_ALL), g/jpeg_data_reader.cc:931.
#include "jpeg_in.h"

#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "jpeg_math.h"
#include "tables.h"

namespace gb200 {

bool JpegInput::is_444() const {
  if (components.size() != 3 || max_h != 1 || max_v != 1) return false;
  for (const JpegComponent& c : components)
    if (c.h_samp != 1 || c.v_samp != 1) return false;
  return true;
}

bool JpegInput::is_420() const {
  return components.size() == 3 && max_h == 2 && max_v == 2 && components[0].h_samp == 2 &&
         components[0].v_samp == 2 && components[1].h_samp == 1 && components[1].v_samp == 1 &&
         components[2].h_samp == 1 && components[2].v_samp == 1;
}

bool has_ycbcr_color_space(const JpegInput& jpg) {
  bool adobe = false;
  uint8_t transform = 0;
  for (const std::string& app : jpg.app_data) {
    const uint8_t marker = static_cast<uint8_t>(app[0]);
    if (marker == 0xe0) return true;  // JFIF
    if (marker == 0xee && app.size() >= 15) {
      adobe = true;
      transform = static_cast<uint8_t>(app[14]);
    }
  }
  if (adobe) return transform != 0;
  return !(jpg.components[0].id == 'R' && jpg.components[1].id == 'G' && jpg.components[2].id == 'B');
}

bool libjpeg_ycbcr(const JpegInput& jpg) {
  bool adobe = false;
  uint8_t transform = 0;
  for (const std::string& app : jpg.app_data) {
    // app: marker byte, two length bytes, payload
    const uint8_t marker = static_cast<uint8_t>(app[0]);
    const size_t payload = app.size() - 3;
    if (marker == 0xe0 && payload >= 14 && app.compare(3, 5, std::string("JFIF\0", 5)) == 0) return true;
    if (marker == 0xee && payload >= 12 && app.compare(3, 5, "Adobe") == 0) {
      adobe = true;
      transform = static_cast<uint8_t>(app[3 + 11]);
    }
  }
  if (adobe) return transform != 0;
  return !(jpg.components[0].id == 'R' && jpg.components[1].id == 'G' && jpg.components[2].id == 'B');
}

bool libjpeg_decodable(const JpegInput& jpg, std::string* why) {
  const int n = static_cast<int>(jpg.components.size());
  if (n == 4) {
    *why = "4 components (CMYK or YCCK): libjpeg gives no RGB or gray output for them";
    return false;
  }
  if (n != 1 && n != 3) {
    *why = std::to_string(n) + " components: libjpeg gives no RGB or gray output for them";
    return false;
  }
  if (n == 3) {
    const JpegComponent* c = jpg.components.data();
    const bool layout = c[0].h_samp == jpg.max_h && c[0].v_samp == jpg.max_v && c[1].h_samp == 1 &&
                        c[1].v_samp == 1 && c[2].h_samp == 1 && c[2].v_samp == 1 &&
                        ((jpg.max_h == 1 && jpg.max_v == 1) || (jpg.max_h == 2 && jpg.max_v == 1) ||
                         (jpg.max_h == 2 && jpg.max_v == 2));
    if (!layout) {
      *why = "sampling factors " + std::to_string(c[0].h_samp) + "x" + std::to_string(c[0].v_samp) + ", " +
             std::to_string(c[1].h_samp) + "x" + std::to_string(c[1].v_samp) + ", " + std::to_string(c[2].h_samp) +
             "x" + std::to_string(c[2].v_samp) + ": only 4:4:4, 4:2:2 and 4:2:0 are decoded";
      return false;
    }
  }
  // smoothing_ok (libjpeg-turbo 2.1 and later, jdcoefct.c): a progressive file is block-smoothed unless
  // some component's DC was never coded, when a coefficient of zig-zag positions 1..9 of some component
  // lacks its last bit (coef_bits != 0: never coded, or coded only down to a bit above 0)
  if (jpg.progressive) {
    bool dc_all = true, useful = false;
    for (int c = 0; c < n && dc_all; ++c) {
      dc_all = jpg.coded_bits[c][0] != 0;
      for (int k = 1; k <= 9; ++k) useful |= (jpg.coded_bits[c][k] & 1) == 0;
    }
    if (dc_all && useful) {
      *why = "progressive file with coefficients not refined to their last bit: libjpeg block-smooths it";
      return false;
    }
  }
  // libjpeg-turbo decodes through its SIMD IDCT where the CPU has one, and that computes libjpeg's
  // integers only within its 16-bit ranges (jpeg_islow).  The exact test runs only on blocks of
  // sum |coef q| > 2040: below that every pass-1 value and sum of them is under 5.66 x 2040 and the
  // output under 2040 / 4 + 1 in magnitude, inside every range.
  for (int c = 0; c < n; ++c) {
    const JpegComponent& comp = jpg.components[c];
    const int* q = jpg.quant[comp.quant_idx].values;
    for (size_t b = 0; b < comp.coeffs.size(); b += 64) {
      const int16_t* blk = &comp.coeffs[b];
      long long t = 0;
      for (int k = 0; k < 64; ++k) t += static_cast<long long>(blk[k] < 0 ? -blk[k] : blk[k]) * q[k];
      if (t > 2040 && !jpeg_islow<true>(blk, q, nullptr, 0)) {
        *why = "coefficients beyond the range in which libjpeg-turbo's SIMD IDCT computes its C IDCT's samples "
               "(component " + std::to_string(c) + ", block " + std::to_string(b / 64) + ")";
        return false;
      }
    }
  }
  return true;
}

bool check_jpeg_sanity(const JpegInput& jpg) {
  for (const JpegComponent& c : jpg.components) {
    const int* q = jpg.quant[c.quant_idx].values;
    for (size_t i = 0; i < c.coeffs.size(); ++i) {
      const long long v = static_cast<long long>(c.coeffs[i]) * q[i & 63];
      if (v > 4096 || v < -4096) return false;
    }
  }
  return true;
}

namespace {

struct Fail {
  std::string* err;
  bool operator()(const char* msg) const {
    if (err) *err = msg;
    fprintf(stderr, "%s\n", msg);
    return false;
  }
};

// Canonical Huffman code of one DHT table: decode by code length.
struct HuffTable {
  bool defined = false;
  int max_code[18];   // largest code of each length, -1 if none
  int val_offset[18]; // index of the first symbol of each length minus its first code
  uint8_t symbols[256];
  int num_symbols = 0;
};

// Segment cursor with bounds checks.
struct Cursor {
  const uint8_t* data;
  size_t len, pos;
  bool have(size_t n) const { return pos + n <= len; }
  int u8() { return data[pos++]; }
  int u16() {
    const int v = (data[pos] << 8) | data[pos + 1];
    pos += 2;
    return v;
  }
};

// MSB-first reader of an entropy-coded segment.  A 0xFF followed by a non-zero byte
// is a marker: the segment ends there and further reads make the scan invalid.  The
// last two bytes of the file are taken to be a marker (EOI) in any case.
class ScanBits {
 public:
  ScanBits(const uint8_t* data, size_t len, size_t pos) : data_(data), len_(len) { restart_at(pos); }
  void restart_at(size_t pos) {
    pos_ = pos;
    acc_ = 0;
    nbits_ = 0;
    stop_ = len_ >= 2 ? len_ - 2 : 0;
    overrun_ = false;
  }
  int bits(int n) {
    if (n == 0) return 0;
    while (nbits_ < n) {
      acc_ = (acc_ << 8) | next_byte();
      nbits_ += 8;
    }
    nbits_ -= n;
    return static_cast<int>((acc_ >> nbits_) & ((1u << n) - 1u));
  }
  int bit() { return bits(1); }
  // Byte position right after the consumed data (pad bits of the last byte dropped);
  // false if the decoder needed bytes beyond the end of the segment.
  bool finish(size_t* pos) {
    nbits_ = 0;
    if (overrun_) return false;
    *pos = pos_;
    return true;
  }

 private:
  unsigned int next_byte() {
    if (pos_ >= stop_) {
      overrun_ = true;
      return 0;
    }
    const unsigned int c = data_[pos_++];
    if (c == 0xff) {
      if (data_[pos_] == 0) {
        ++pos_;  // stuffed zero
      } else {
        // that 0xFF starts a marker: it was not data
        stop_ = pos_ - 1;
        pos_ = stop_;
        overrun_ = true;
        return 0;
      }
    }
    return c;
  }
  const uint8_t* data_;
  size_t len_, pos_, stop_;
  uint64_t acc_;
  int nbits_;
  bool overrun_;
};

int decode_symbol(const HuffTable& t, ScanBits* br) {
  int code = 0;
  for (int l = 1; l <= 16; ++l) {
    code = (code << 1) | br->bit();
    if (t.max_code[l] >= 0 && code <= t.max_code[l]) {
      const int idx = t.val_offset[l] + code;
      return idx < t.num_symbols ? t.symbols[idx] : -1;
    }
  }
  return -1;
}

inline int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

struct ScanSpec {
  int ncomp;
  int comp[4], dc_tbl[4], ac_tbl[4];
  int ss, se, ah, al;
};

class Reader {
 public:
  Reader(const uint8_t* data, size_t len, JpegInput* jpg, std::string* err) : c_{data, len, 0}, jpg_(jpg), fail_{err} {
    memset(progression_, 0, sizeof(progression_));
  }

  bool run() {
    if (!c_.have(2) || c_.data[0] != 0xff || c_.data[1] != 0xd8) return fail_("Did not find expected SOI marker");
    c_.pos = 2;
    int marker = 0;
    do {
      skip_to_marker();
      if (!c_.have(2) || c_.data[c_.pos] != 0xff) return fail_("Marker byte (0xff) expected");
      marker = c_.data[c_.pos + 1];
      c_.pos += 2;
      bool ok = true;
      if (marker == 0xc0 || marker == 0xc1 || marker == 0xc2) {
        progressive_ = marker == 0xc2;
        ok = frame_header();
      } else if (marker == 0xc4) {
        ok = huffman_tables();
      } else if (marker >= 0xd0 && marker <= 0xd7) {
        // stray restart marker: no payload
      } else if (marker == 0xd9) {
        // end of image
      } else if (marker == 0xda) {
        ok = scan();
      } else if (marker == 0xdb) {
        ok = quant_tables();
      } else if (marker == 0xdd) {
        ok = restart_interval();
      } else if (marker >= 0xe0 && marker <= 0xef) {
        ok = keep_segment(&jpg_->app_data, 3);
      } else if (marker == 0xfe) {
        ok = keep_segment(&jpg_->com_data, 2);
      } else {
        ok = fail_("Unsupported marker");
      }
      if (!ok) return false;
    } while (marker != 0xd9);
    if (!have_frame_) return fail_("Missing SOF marker.");
    if (c_.pos < c_.len) jpg_->tail_data.assign(reinterpret_cast<const char*>(c_.data + c_.pos), c_.len - c_.pos);
    // component Tq -> position of that table in the list (first match)
    for (JpegComponent& comp : jpg_->components) {
      int found = -1;
      for (size_t j = 0; j < jpg_->quant.size() && found < 0; ++j)
        if (jpg_->quant[j].index == comp.quant_idx) found = static_cast<int>(j);
      if (found < 0) return fail_("Quantization table not found");
      comp.quant_idx = found;
    }
    if (num_dht_ == 0) return fail_("Need at least one Huffman code table.");
    if (num_dht_ >= 512) return fail_("Too many Huffman tables.");
    jpg_->progressive = progressive_;
    memcpy(jpg_->coded_bits, progression_, sizeof(progression_));
    return true;
  }

 private:
  // Bytes between segments that are not a marker the format knows are skipped.
  void skip_to_marker() {
    static const uint8_t kKnown[64] = {
        1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 0, 1, 0, 0,
        1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0};
    while (c_.pos + 1 < c_.len) {
      const uint8_t* p = c_.data + c_.pos;
      if (p[0] == 0xff && p[1] >= 0xc0 && kKnown[p[1] - 0xc0]) break;
      ++c_.pos;
    }
  }

  bool segment_end(size_t start, size_t marker_len) {
    if (start + marker_len != c_.pos) return fail_("Invalid marker length");
    return true;
  }

  bool frame_header() {
    if (have_frame_) return fail_("Duplicate SOF marker.");
    have_frame_ = true;
    const size_t start = c_.pos;
    if (!c_.have(8)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    const int precision = c_.u8(), height = c_.u16(), width = c_.u16(), ncomp = c_.u8();
    if (precision != 8) return fail_("Invalid precision");
    if (height < 1 || width < 1) return fail_("Invalid image size");
    if (ncomp < 1 || ncomp > 4) return fail_("Invalid number of components");
    if (!c_.have(3 * static_cast<size_t>(ncomp))) return fail_("Unexpected end of input");
    jpg_->width = width;
    jpg_->height = height;
    jpg_->components.resize(ncomp);
    bool seen[256] = {false};
    for (JpegComponent& comp : jpg_->components) {
      comp.id = c_.u8();
      if (seen[comp.id]) return fail_("Duplicate ID in SOF.");
      seen[comp.id] = true;
      const int f = c_.u8();
      comp.h_samp = f >> 4;
      comp.v_samp = f & 15;
      if (comp.h_samp < 1 || comp.v_samp < 1) return fail_("Invalid sampling factor");
      comp.quant_idx = c_.u8();
      jpg_->max_h = std::max(jpg_->max_h, comp.h_samp);
      jpg_->max_v = std::max(jpg_->max_v, comp.v_samp);
    }
    jpg_->mcu_rows = (height + 8 * jpg_->max_v - 1) / (8 * jpg_->max_v);
    jpg_->mcu_cols = (width + 8 * jpg_->max_h - 1) / (8 * jpg_->max_h);
    for (JpegComponent& comp : jpg_->components) {
      if (jpg_->max_h % comp.h_samp != 0 || jpg_->max_v % comp.v_samp != 0)
        return fail_("Non-integral subsampling ratios.");
      comp.width_in_blocks = jpg_->mcu_cols * comp.h_samp;
      comp.height_in_blocks = jpg_->mcu_rows * comp.v_samp;
      const uint64_t nb = static_cast<uint64_t>(comp.width_in_blocks) * comp.height_in_blocks;
      if (nb > (1ull << 21)) return fail_("Image too large.");
      comp.coeffs.assign(static_cast<size_t>(nb) * 64, 0);
    }
    return segment_end(start, marker_len);
  }

  bool quant_tables() {
    const size_t start = c_.pos;
    if (!c_.have(2)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    if (marker_len == 2) return fail_("DQT marker: no quantization table found");
    const int* zz = zigzag_to_natural();
    while (c_.pos < start + marker_len && jpg_->quant.size() < 4) {
      if (!c_.have(1)) return fail_("Unexpected end of input");
      const int pq_tq = c_.u8();
      JpegQuantTable t;
      t.precision = pq_tq >> 4;
      t.index = pq_tq & 15;
      if (t.index > 3) return fail_("Invalid quantization table index");
      if (!c_.have((t.precision ? 2 : 1) * 64)) return fail_("Unexpected end of input");
      for (int k = 0; k < 64; ++k) {
        const int v = t.precision ? c_.u16() : c_.u8();
        if (v < 1) return fail_("Invalid quantization value");
        t.values[zz[k]] = v;
      }
      jpg_->quant.push_back(t);
    }
    return segment_end(start, marker_len);
  }

  bool huffman_tables() {
    const size_t start = c_.pos;
    if (!c_.have(2)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    if (marker_len == 2) return fail_("DHT marker: no Huffman table found");
    while (c_.pos < start + marker_len) {
      if (!c_.have(17)) return fail_("Unexpected end of input");
      const int tc_th = c_.u8();
      const bool ac = (tc_th & 0x10) != 0;
      const int slot = tc_th & 0x0f;
      if ((tc_th & 0xe0) != 0 || slot > 3) return fail_("Invalid Huffman table index");
      HuffTable& t = ac ? ac_[slot] : dc_[slot];
      int counts[17] = {0};
      int total = 0;
      long space = 1L << 16;
      int longest = 1;
      for (int l = 1; l <= 16; ++l) {
        counts[l] = c_.u8();
        if (counts[l]) longest = l;
        total += counts[l];
        space -= static_cast<long>(counts[l]) << (16 - l);
      }
      if (total > (ac ? 256 : 12)) return fail_("Invalid Huffman code");
      if (!c_.have(total)) return fail_("Unexpected end of input");
      bool seen[256] = {false};
      for (int i = 0; i < total; ++i) {
        const int v = c_.u8();
        if (!ac && v > 11) return fail_("Invalid Huffman code value");
        if (seen[v]) return fail_("Duplicate Huffman code value");
        seen[v] = true;
        t.symbols[i] = static_cast<uint8_t>(v);
      }
      // the all-ones code of the longest length must stay free
      space -= 1L << (16 - longest);
      if (space < 0) return fail_("Invalid Huffman code lengths.");
      t.num_symbols = total;
      int code = 0, k = 0;
      for (int l = 1; l <= 16; ++l) {
        t.val_offset[l] = k - code;
        k += counts[l];
        code += counts[l];
        t.max_code[l] = counts[l] ? code - 1 : -1;
        code <<= 1;
      }
      t.defined = true;
      ++num_dht_;
    }
    return segment_end(start, marker_len);
  }

  bool restart_interval() {
    if (restart_interval_ > 0) return fail_("Duplicate DRI marker.");
    const size_t start = c_.pos;
    if (!c_.have(4)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    restart_interval_ = c_.u16();
    return segment_end(start, marker_len);
  }

  // `back` = how many bytes before the payload belong to the kept string (APPn keeps
  // its marker byte and the length, COM only the length).
  bool keep_segment(std::vector<std::string>* list, int back) {
    if (!c_.have(2)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    if (marker_len < 2) return fail_("Invalid marker length");
    if (!c_.have(marker_len - 2)) return fail_("Unexpected end of input");
    list->push_back(std::string(reinterpret_cast<const char*>(c_.data + c_.pos - back), marker_len + back - 2));
    c_.pos += marker_len - 2;
    return true;
  }

  bool scan_header(ScanSpec* s) {
    const size_t start = c_.pos;
    if (!c_.have(3)) return fail_("Unexpected end of input");
    const size_t marker_len = c_.u16();
    s->ncomp = c_.u8();
    if (s->ncomp < 1 || s->ncomp > static_cast<int>(jpg_->components.size()))
      return fail_("Invalid number of components in scan");
    if (!c_.have(2 * static_cast<size_t>(s->ncomp))) return fail_("Unexpected end of input");
    bool seen[256] = {false};
    for (int i = 0; i < s->ncomp; ++i) {
      const int id = c_.u8();
      if (seen[id]) return fail_("Duplicate ID in SOS.");
      seen[id] = true;
      int idx = -1;
      for (size_t j = 0; j < jpg_->components.size(); ++j)
        if (jpg_->components[j].id == id) idx = static_cast<int>(j);
      if (idx < 0) return fail_("SOS marker: Could not find component");
      s->comp[i] = idx;
      const int t = c_.u8();
      s->dc_tbl[i] = t >> 4;
      s->ac_tbl[i] = t & 15;
      if (s->dc_tbl[i] > 3 || s->ac_tbl[i] > 3) return fail_("Invalid Huffman table index");
    }
    if (!c_.have(3)) return fail_("Unexpected end of input");
    s->ss = c_.u8();
    s->se = c_.u8();
    if (s->ss > 63 || s->se < s->ss || s->se > 63) return fail_("Invalid spectral selection");
    const int a = c_.u8();
    s->ah = a >> 4;
    s->al = a & 15;
    for (int i = 0; i < s->ncomp; ++i) {
      if (s->ss == 0 && !dc_[s->dc_tbl[i]].defined) return fail_("SOS marker: Could not find DC Huffman table");
      if (s->se > 0 && !ac_[s->ac_tbl[i]].defined) return fail_("SOS marker: Could not find AC Huffman table");
    }
    return segment_end(start, marker_len);
  }

  // First pass over a band of one block (sequential data, or a progressive scan with
  // Ah = 0): DC difference, then run/size coded AC values, shifted left by Al.
  bool first_pass(const ScanSpec& s, int i, int ss, int se, int al, ScanBits* br, int* last_dc, int16_t* blk) {
    const int* zz = zigzag_to_natural();
    const bool band_has_no_dc = ss > 0;
    if (ss == 0) {
      int sz = decode_symbol(dc_[s.dc_tbl[i]], br);
      if (sz < 0 || sz > 11) return fail_("Invalid Huffman symbol for DC coefficient.");
      int diff = 0;
      if (sz > 0) diff = extend(br->bits(sz), sz);
      diff += *last_dc;
      const int v = diff * (1 << al);
      blk[0] = static_cast<int16_t>(v);
      if (blk[0] != v) return fail_("Invalid DC coefficient");
      *last_dc = diff;
      ++ss;
    }
    if (ss > se) return true;
    if (eobrun_ > 0) {
      --eobrun_;
      return true;
    }
    const HuffTable& act = ac_[s.ac_tbl[i]];
    for (int k = ss; k <= se; ++k) {
      const int sym = decode_symbol(act, br);
      if (sym < 0) return fail_("Invalid Huffman symbol for AC coefficient");
      const int run = sym >> 4, sz = sym & 15;
      if (sz > 0) {
        k += run;
        if (k > se) return fail_("Out-of-band coefficient");
        if (sz + al >= 12) return fail_("Out of range AC coefficient value");
        blk[zz[k]] = static_cast<int16_t>(extend(br->bits(sz), sz) * (1 << al));
      } else if (run == 15) {
        k += 15;
      } else {
        eobrun_ = 1 << run;
        if (run > 0) {
          if (!band_has_no_dc) return fail_("End-of-block run crossing DC coeff.");
          eobrun_ += br->bits(run);
        }
        break;
      }
    }
    --eobrun_;
    return true;
  }

  // One correction bit for an already non-zero coefficient (T.81 G.1.2.3).
  static void correct(int16_t* c, int bit, int plus, int minus) {
    if (bit && (*c & plus) == 0) *c = static_cast<int16_t>(*c + (*c >= 0 ? plus : minus));
  }

  // Successive-approximation refinement of a band (Ah > 0).
  bool refine_pass(const ScanSpec& s, int i, int ss, int se, int al, ScanBits* br, int16_t* blk) {
    const int* zz = zigzag_to_natural();
    const bool band_has_no_dc = ss > 0;
    if (ss == 0) {
      blk[0] = static_cast<int16_t>(blk[0] | (br->bit() << al));
      ++ss;
    }
    if (ss > se) return true;
    const int plus = 1 << al, minus = -(1 << al);
    const HuffTable& act = ac_[s.ac_tbl[i]];
    int k = ss;
    bool open_zero_run = false;
    if (eobrun_ <= 0) {
      for (; k <= se; ++k) {
        const int sym = decode_symbol(act, br);
        if (sym < 0) return fail_("Invalid Huffman symbol for AC coefficient");
        int run = sym >> 4;
        const int sz = sym & 15;
        int newval = 0;
        if (sz != 0) {
          if (sz != 1) return fail_("Invalid Huffman symbol for AC coefficient");
          newval = br->bit() ? plus : minus;
          open_zero_run = false;
        } else if (run != 15) {
          eobrun_ = 1 << run;
          if (run > 0) {
            if (!band_has_no_dc) return fail_("End-of-block run crossing DC coeff.");
            eobrun_ += br->bits(run);
          }
          break;
        } else {
          open_zero_run = true;
        }
        // pass over `run` zero-history coefficients, correcting the non-zero ones met on the way
        while (k <= se) {
          int16_t* c = &blk[zz[k]];
          if (*c != 0) {
            correct(c, br->bit(), plus, minus);
          } else if (--run < 0) {
            break;
          }
          ++k;
        }
        if (newval) {
          if (k > se) return fail_("Out-of-band coefficient");
          blk[zz[k]] = static_cast<int16_t>(newval);
        }
      }
    }
    if (open_zero_run) return fail_("Extra zero run before end-of-block.");
    if (eobrun_ > 0) {
      for (; k <= se; ++k) {
        int16_t* c = &blk[zz[k]];
        if (*c != 0) correct(c, br->bit(), plus, minus);
      }
    }
    --eobrun_;
    return true;
  }

  bool scan() {
    ScanSpec s;
    if (!scan_header(&s)) return false;
    const bool interleaved = s.ncomp > 1;
    int mcus_per_row = jpg_->mcu_cols, mcu_rows = jpg_->mcu_rows;
    if (!interleaved) {
      const JpegComponent& comp = jpg_->components[s.comp[0]];
      mcus_per_row = (jpg_->width * comp.h_samp + 8 * jpg_->max_h - 1) / (8 * jpg_->max_h);
      mcu_rows = (jpg_->height * comp.v_samp + 8 * jpg_->max_v - 1) / (8 * jpg_->max_v);
    }
    const int al = progressive_ ? s.al : 0, ah = progressive_ ? s.ah : 0;
    const int ss = progressive_ ? s.ss : 0, se = progressive_ ? s.se : 63;
    // every (component, coefficient) bit may be coded once, coarse bits first
    const unsigned int mask = (ah == 0 ? (0xffffu << al) : (1u << al)) & 0xffffu;
    const unsigned int finer = (1u << al) - 1u;
    for (int i = 0; i < s.ncomp; ++i)
      for (int k = ss; k <= se; ++k) {
        uint16_t& p = progression_[s.comp[i]][k];
        if (p & mask) return fail_("Overlapping scans");
        if (p & finer) return fail_("Invalid scan order, a more refined scan was already done");
        p = static_cast<uint16_t>(p | mask);
      }
    if (al > 10) return fail_("Scan parameter Al is not supported in guetzli.");

    ScanBits br(c_.data, c_.len, c_.pos);
    int last_dc[4] = {0, 0, 0, 0};
    int to_go = restart_interval_, next_rst = 0;
    eobrun_ = -1;
    for (int my = 0; my < mcu_rows; ++my) {
      for (int mx = 0; mx < mcus_per_row; ++mx) {
        if (restart_interval_ > 0) {
          if (to_go == 0) {
            size_t p = 0;
            if (!br.finish(&p)) return fail_("Unexpected end of scan.");
            if (p + 2 > c_.len || c_.data[p] != 0xff) return fail_("Marker byte (0xff) expected");
            if (c_.data[p + 1] != 0xd0 + next_rst) return fail_("Did not find expected restart marker");
            br.restart_at(p + 2);
            next_rst = (next_rst + 1) & 7;
            to_go = restart_interval_;
            memset(last_dc, 0, sizeof(last_dc));
            if (eobrun_ > 0) return fail_("End-of-block run too long.");
            eobrun_ = -1;
          }
          --to_go;
        }
        for (int i = 0; i < s.ncomp; ++i) {
          JpegComponent& comp = jpg_->components[s.comp[i]];
          const int nby = interleaved ? comp.v_samp : 1, nbx = interleaved ? comp.h_samp : 1;
          for (int iy = 0; iy < nby; ++iy)
            for (int ix = 0; ix < nbx; ++ix) {
              const int by = my * nby + iy, bx = mx * nbx + ix;
              int16_t* blk = &comp.coeffs[(static_cast<size_t>(by) * comp.width_in_blocks + bx) * 64];
              const bool ok = ah == 0 ? first_pass(s, i, ss, se, al, &br, &last_dc[s.comp[i]], blk)
                                      : refine_pass(s, i, ss, se, al, &br, blk);
              if (!ok) return false;
            }
        }
      }
    }
    if (eobrun_ > 0) return fail_("End-of-block run too long.");
    size_t p = 0;
    if (!br.finish(&p)) return fail_("Unexpected end of scan.");
    if (p > c_.len) return fail_("Unexpected end of file during scan.");
    c_.pos = p;
    return true;
  }

  Cursor c_;
  JpegInput* jpg_;
  Fail fail_;
  HuffTable dc_[4], ac_[4];
  uint16_t progression_[4][64];
  bool progressive_ = false, have_frame_ = false;
  int restart_interval_ = 0, num_dht_ = 0, eobrun_ = -1;
};

}  // namespace

bool read_jpeg_dimensions(const uint8_t* data, size_t len, int* width, int* height) {
  if (len < 4 || data[0] != 0xff || data[1] != 0xd8) return false;
  size_t pos = 2;
  while (pos + 4 <= len) {
    if (data[pos] != 0xff) {  // tolerate filler between segments like the full reader
      ++pos;
      continue;
    }
    const int marker = data[pos + 1];
    if (marker == 0xff || marker == 0x00 || (marker >= 0xd0 && marker <= 0xd7)) {
      pos += marker == 0xff ? 1 : 2;
      continue;
    }
    if (marker == 0xd9 || marker == 0xda) return false;  // image data before any frame header
    const size_t seg = (static_cast<size_t>(data[pos + 2]) << 8) | data[pos + 3];
    if (seg < 2 || pos + 2 + seg > len) return false;
    if (marker == 0xc0 || marker == 0xc1 || marker == 0xc2) {
      if (seg < 8 || data[pos + 4] != 8) return false;
      *height = (data[pos + 5] << 8) | data[pos + 6];
      *width = (data[pos + 7] << 8) | data[pos + 8];
      return *height >= 1 && *width >= 1;
    }
    pos += 2 + seg;
  }
  return false;
}

bool read_jpeg(const uint8_t* data, size_t len, JpegInput* jpg, std::string* err) {
  *jpg = JpegInput();
  Reader r(data, len, jpg, err);
  return r.run();
}

}  // namespace gb200
