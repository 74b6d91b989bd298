// run_OF_INT / run_OF_RGB / run_DE_INT / run_DE_RGB -- command-line drop-in for the
// reference binaries (argument grammar and TIME lines of run_dense.cpp:185-431,
// README.md:48-88), built on the CUDA hot path through OFC::OFClass (ofdis_host.h).
//
//   run_*_* image1 image2 outputfile [oppoint | p1 .. p20]
//
// No OpenCV: images are read by a small built-in decoder (binary PGM/PPM, and
// 8-bit non-interlaced PNG through zlib); pyramid, Sobel/8 gradients, padding,
// x2^lv_l upsampling, crop and .flo/.pfm writing restate run_dense.cpp:130-178,
// 298-344,384-421 (exact for 8-bit input, see of_dis_b200/preprocess.py).
// SELECTMODE 1 = optical flow, 2 = stereo; SELECTCHANNEL 1 = gray, 3 = RGB
// (CMakeLists.txt:25-46).
#include <sys/time.h>
#include <zlib.h>

#include <cfloat>
#include <cstdarg>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "ofdis_host.h"

#ifndef SELECTMODE
#define SELECTMODE 1
#endif
#ifndef SELECTCHANNEL
#define SELECTCHANNEL 1
#endif

using namespace std;

namespace {

struct Image8 {
  int w = 0, h = 0, c = 0;  // c channels, interleaved; colour order B,G,R like cv::imread
  vector<uint8_t> px;
};

bool read_file(const char* path, vector<uint8_t>& buf) {
  FILE* f = fopen(path, "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  buf.resize(n > 0 ? n : 0);
  size_t got = n > 0 ? fread(buf.data(), 1, n, f) : 0;
  fclose(f);
  return (long)got == n && n > 0;
}

// ---- binary PNM -------------------------------------------------------------
bool decode_pnm(const vector<uint8_t>& b, Image8& im, vector<uint8_t>& rgb, int& ch) {
  if (b.size() < 3 || b[0] != 'P' || (b[1] != '5' && b[1] != '6')) return false;
  ch = b[1] == '5' ? 1 : 3;
  size_t pos = 2;
  int vals[3], nv = 0;
  while (nv < 3 && pos < b.size()) {
    while (pos < b.size() && isspace(b[pos])) ++pos;
    if (pos < b.size() && b[pos] == '#') {
      while (pos < b.size() && b[pos] != '\n') ++pos;
      continue;
    }
    int v = 0, d = 0;
    while (pos < b.size() && isdigit(b[pos])) {
      if (++d > 6) return false;  // no header number has more than 6 digits: no int overflow
      v = v * 10 + (b[pos++] - '0');
    }
    if (!d) return false;
    vals[nv++] = v;
  }
  ++pos;  // single whitespace after maxval
  if (nv < 3 || vals[2] != 255 || vals[0] <= 0 || vals[1] <= 0 || vals[0] > (1 << 15) || vals[1] > (1 << 15)) return false;
  im.w = vals[0];
  im.h = vals[1];
  const size_t n = (size_t)im.w * im.h * ch;
  if (pos + n > b.size()) return false;
  rgb.assign(b.begin() + pos, b.begin() + pos + n);
  return true;
}

// ---- PNG (8-bit, colour types 0,2,3,4,6, non-interlaced) ----------------------
uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; }

bool decode_png(const vector<uint8_t>& b, Image8& im, vector<uint8_t>& rgb, int& ch) {
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (b.size() < 8 || memcmp(b.data(), sig, 8)) return false;
  size_t pos = 8;
  int depth = 0, ctype = 0, interlace = 0;
  vector<uint8_t> idat, plte;
  while (pos + 8 <= b.size()) {
    const uint32_t len = be32(&b[pos]);
    const char* type = (const char*)&b[pos + 4];
    const uint8_t* data = &b[pos + 8];
    if (pos + 12 + len > b.size()) return false;
    if (!memcmp(type, "IHDR", 4)) {
      if (len < 13) return false;
      im.w = be32(data);
      im.h = be32(data + 4);
      depth = data[8];
      ctype = data[9];
      interlace = data[12];
    } else if (!memcmp(type, "PLTE", 4)) plte.assign(data, data + len);
    else if (!memcmp(type, "IDAT", 4)) idat.insert(idat.end(), data, data + len);
    else if (!memcmp(type, "IEND", 4)) break;
    pos += 12 + len;
  }
  if (depth != 8 || interlace != 0 || im.w <= 0 || im.h <= 0 || im.w > (1 << 15) || im.h > (1 << 15)) return false;
  int spp;  // samples per pixel in the file
  switch (ctype) {
    case 0: spp = 1; break;
    case 2: spp = 3; break;
    case 3: spp = 1; break;
    case 4: spp = 2; break;
    case 6: spp = 4; break;
    default: return false;
  }
  const size_t stride = (size_t)im.w * spp;
  vector<uint8_t> raw((stride + 1) * im.h);
  uLongf rawlen = raw.size();
  if (uncompress(raw.data(), &rawlen, idat.data(), idat.size()) != Z_OK || rawlen != raw.size()) return false;
  vector<uint8_t> img(stride * im.h), zero(stride, 0);
  for (int y = 0; y < im.h; ++y) {
    const uint8_t ft = raw[(stride + 1) * y];
    const uint8_t* in = &raw[(stride + 1) * y + 1];
    uint8_t* out = &img[stride * y];
    const uint8_t* up = y ? &img[stride * (y - 1)] : zero.data();
    for (size_t x = 0; x < stride; ++x) {
      const int a = x >= (size_t)spp ? out[x - spp] : 0, bb = up[x], c = x >= (size_t)spp ? up[x - spp] : 0;
      int pr = 0;
      switch (ft) {
        case 0: pr = 0; break;
        case 1: pr = a; break;
        case 2: pr = bb; break;
        case 3: pr = (a + bb) >> 1; break;
        case 4: {
          const int p = a + bb - c, pa = abs(p - a), pb = abs(p - bb), pc = abs(p - c);
          pr = (pa <= pb && pa <= pc) ? a : (pb <= pc ? bb : c);
          break;
        }
        default: return false;
      }
      out[x] = (uint8_t)(in[x] + pr);
    }
  }
  ch = (ctype == 0 || ctype == 4) ? 1 : 3;
  rgb.resize((size_t)im.w * im.h * ch);
  for (size_t i = 0; i < (size_t)im.w * im.h; ++i) {
    const uint8_t* s = &img[i * spp];
    if (ctype == 0 || ctype == 4) rgb[i] = s[0];
    else if (ctype == 3) {
      if ((size_t)s[0] * 3 + 3 > plte.size()) return false;  // palette index beyond PLTE
      const uint8_t* e = &plte[(size_t)s[0] * 3];
      rgb[i * 3] = e[0]; rgb[i * 3 + 1] = e[1]; rgb[i * 3 + 2] = e[2];
    } else {
      rgb[i * 3] = s[0]; rgb[i * 3 + 1] = s[1]; rgb[i * 3 + 2] = s[2];
    }
  }
  return true;
}

// cv::imread semantics: COLOR -> BGR; GRAYSCALE -> 1 channel.  A colour PNM goes through cvtColor's
// 14-bit BT.601 fixed point, a colour PNG through libpng's png_set_rgb_to_gray(0.299, 0.587): 15-bit
// coefficients 9797 / 19234 / 3737, truncating (checked against cv2 4.13: both formulas reproduce
// cv2.imread(..., IMREAD_GRAYSCALE) exactly on random colour images, tests/test_params_io.py).
bool load_image(const char* path, int want_channels, Image8& im) {
  vector<uint8_t> file, rgb;
  int ch = 0;
  if (!read_file(path, file)) return false;
  bool from_png = false;
  try {
    if (!decode_pnm(file, im, rgb, ch)) {
      if (!decode_png(file, im, rgb, ch)) return false;
      from_png = true;
    }
  } catch (const std::exception&) {  // bad_alloc / length errors on malformed headers
    return false;
  }
  im.c = want_channels;
  const size_t n = (size_t)im.w * im.h;
  im.px.resize(n * want_channels);
  for (size_t i = 0; i < n; ++i) {
    if (want_channels == 1) {
      if (ch == 1) im.px[i] = rgb[i];
      else {
        const int r = rgb[i * 3], g = rgb[i * 3 + 1], b = rgb[i * 3 + 2];
        im.px[i] = from_png ? (uint8_t)((r * 9797 + g * 19234 + b * 3737) >> 15)
                            : (uint8_t)((r * 4899 + g * 9617 + b * 1868 + 8192) >> 14);
      }
    } else {
      if (ch == 1) im.px[i * 3] = im.px[i * 3 + 1] = im.px[i * 3 + 2] = rgb[i];
      else { im.px[i * 3] = rgb[i * 3 + 2]; im.px[i * 3 + 1] = rgb[i * 3 + 1]; im.px[i * 3 + 2] = rgb[i * 3]; }
    }
  }
  return true;
}

// ---- float images ---------------------------------------------------------------
struct ImageF {
  int w = 0, h = 0, c = 1;
  vector<float> px;
  float& at(int x, int y, int k) { return px[((size_t)y * w + x) * c + k]; }
  float at(int x, int y, int k) const { return px[((size_t)y * w + x) * c + k]; }
};

int clampi(int v, int n) { return v < 0 ? 0 : (v > n - 1 ? n - 1 : v); }
int reflect101(int v, int n) {
  if (n == 1) return 0;
  while (v < 0 || v >= n) v = v < 0 ? -v : 2 * (n - 1) - v;
  return v;
}

// copyMakeBorder: replicate (image) or constant zero (gradients)
ImageF pad(const ImageF& s, int t, int b, int l, int r, bool replicate) {
  ImageF d;
  d.w = s.w + l + r;
  d.h = s.h + t + b;
  d.c = s.c;
  d.px.assign((size_t)d.w * d.h * d.c, 0.f);
  for (int y = 0; y < d.h; ++y)
    for (int x = 0; x < d.w; ++x) {
      const int sx = x - l, sy = y - t;
      if (!replicate && (sx < 0 || sy < 0 || sx >= s.w || sy >= s.h)) continue;
      for (int k = 0; k < s.c; ++k) d.at(x, y, k) = s.at(clampi(sx, s.w), clampi(sy, s.h), k);
    }
  return d;
}

// cv::resize(.5,.5,INTER_LINEAR) on even sizes (run_dense.cpp:150)
ImageF half_size(const ImageF& s) {
  ImageF d;
  d.w = s.w / 2;
  d.h = s.h / 2;
  d.c = s.c;
  d.px.resize((size_t)d.w * d.h * d.c);
  for (int y = 0; y < d.h; ++y)
    for (int x = 0; x < d.w; ++x)
      for (int k = 0; k < s.c; ++k)
        d.at(x, y, k) = ((s.at(2 * x, 2 * y, k) + s.at(2 * x + 1, 2 * y, k)) +
                         (s.at(2 * x, 2 * y + 1, k) + s.at(2 * x + 1, 2 * y + 1, k))) * 0.25f;
  return d;
}

// cv::Sobel(CV_32F, 3x3, scale 1/8, BORDER_DEFAULT) (run_dense.cpp:156-157)
void sobel8(const ImageF& s, ImageF& dx, ImageF& dy) {
  dx = s;
  dy = s;
  for (int y = 0; y < s.h; ++y)
    for (int x = 0; x < s.w; ++x)
      for (int k = 0; k < s.c; ++k) {
        const int xm = reflect101(x - 1, s.w), xp = reflect101(x + 1, s.w), ym = reflect101(y - 1, s.h),
                  yp = reflect101(y + 1, s.h);
        const float t0 = s.at(xp, ym, k) - s.at(xm, ym, k), t1 = s.at(xp, y, k) - s.at(xm, y, k),
                    t2 = s.at(xp, yp, k) - s.at(xm, yp, k);
        dx.at(x, y, k) = (t0 * 0.125f + t1 * 0.25f) + t2 * 0.125f;
        const float s0 = (s.at(xm, ym, k) * 0.125f + s.at(x, ym, k) * 0.25f) + s.at(xp, ym, k) * 0.125f;
        const float s2 = (s.at(xm, yp, k) * 0.125f + s.at(x, yp, k) * 0.25f) + s.at(xp, yp, k) * 0.125f;
        dy.at(x, y, k) = s2 - s0;
      }
}

// ConstructImgPyramide (run_dense.cpp:130-178)
void ConstructImgPyramide(const ImageF& img, vector<ImageF>& pyr, vector<ImageF>& pyr_dx, vector<ImageF>& pyr_dy,
                          const float** img_pyr, const float** dx_pyr, const float** dy_pyr, int lv_f,
                          int imgpadding) {
  pyr.resize(lv_f + 1);
  pyr_dx.resize(lv_f + 1);
  pyr_dy.resize(lv_f + 1);
  for (int i = 0; i <= lv_f; ++i) {
    pyr[i] = i == 0 ? img : half_size(pyr[i - 1]);
    sobel8(pyr[i], pyr_dx[i], pyr_dy[i]);
  }
  for (int i = 0; i <= lv_f; ++i) {
    pyr[i] = pad(pyr[i], imgpadding, imgpadding, imgpadding, imgpadding, true);
    pyr_dx[i] = pad(pyr_dx[i], imgpadding, imgpadding, imgpadding, imgpadding, false);
    pyr_dy[i] = pad(pyr_dy[i], imgpadding, imgpadding, imgpadding, imgpadding, false);
    img_pyr[i] = pyr[i].px.data();
    dx_pyr[i] = pyr_dx[i].px.data();
    dy_pyr[i] = pyr_dy[i].px.data();
  }
}

int AutoFirstScaleSelect(int imgwidth, int fratio, int patchsize) {  // run_dense.cpp:180-183
  return std::max(0, (int)std::floor(log2((2.0f * (float)imgwidth) / ((float)fratio * (float)patchsize))));
}

// cv::resize(fx=fy=s, INTER_LINEAR): src = (dst+.5)/s-.5, clamped (run_dense.cpp:410)
ImageF upsample_linear(const ImageF& s, int sc) {
  ImageF d;
  d.w = s.w * sc;
  d.h = s.h * sc;
  d.c = s.c;
  d.px.resize((size_t)d.w * d.h * d.c);
  auto taps = [&](int n_src, int n_dst, vector<int>& i0, vector<int>& i1, vector<float>& f) {
    i0.resize(n_dst); i1.resize(n_dst); f.resize(n_dst);
    for (int x = 0; x < n_dst; ++x) {
      const float fx = ((float)x + 0.5f) / (float)sc - 0.5f;
      const int x0 = (int)floorf(fx);
      f[x] = x0 < 0 ? 0.f : fx - (float)x0;
      i0[x] = clampi(x0, n_src);
      i1[x] = clampi(x0 + 1, n_src);
    }
  };
  vector<int> x0, x1, y0, y1;
  vector<float> fx, fy;
  taps(s.w, d.w, x0, x1, fx);
  taps(s.h, d.h, y0, y1, fy);
  ImageF rows;
  rows.w = d.w; rows.h = s.h; rows.c = s.c;
  rows.px.resize((size_t)rows.w * rows.h * rows.c);
  for (int y = 0; y < s.h; ++y)
    for (int x = 0; x < d.w; ++x)
      for (int k = 0; k < s.c; ++k)
        rows.at(x, y, k) = s.at(x0[x], y, k) * (1.0f - fx[x]) + s.at(x1[x], y, k) * fx[x];
  for (int y = 0; y < d.h; ++y)
    for (int x = 0; x < d.w; ++x)
      for (int k = 0; k < s.c; ++k)
        d.at(x, y, k) = rows.at(x, y0[y], k) * (1.0f - fy[y]) + rows.at(x, y1[y], k) * fy[y];
  return d;
}

// SaveFlowFile (run_dense.cpp:16-57)
void SaveFlowFile(const ImageF& img, const char* filename) {
  FILE* stream = fopen(filename, "wb");
  if (stream == 0) {
    cout << "WriteFile: could not open file" << endl;
    return;
  }
  fprintf(stream, "PIEH");
  if ((int)fwrite(&img.w, sizeof(int), 1, stream) != 1 || (int)fwrite(&img.h, sizeof(int), 1, stream) != 1)
    cout << "WriteFile: problem writing header" << endl;
  if (fwrite(img.px.data(), sizeof(float), img.px.size(), stream) != img.px.size())
    cout << "WriteFile: problem writing data" << endl;
  fclose(stream);
}

// SavePFMFile (run_dense.cpp:60-81)
void SavePFMFile(const ImageF& img, const char* filename) {
  FILE* stream = fopen(filename, "wb");
  if (stream == 0) {
    cout << "WriteFile: could not open file" << endl;
    return;
  }
  fprintf(stream, "Pf\n%d %d\n%f\n", img.w, img.h, (float)-1.0f);
  for (int y = img.h - 1; y >= 0; --y)
    for (int x = 0; x < img.w; ++x) {
      float tmp = -img.at(x, y, 0);
      if ((int)fwrite(&tmp, sizeof(float), 1, stream) != 1) cout << "WriteFile: problem writing data" << endl;
    }
  fclose(stream);
}

// A flow file of the image size: the init flow of the reference's commented-out input (run_dense.cpp:292-293,355-378)
// or the ground truth of run_*_batch --gt, checked before any device work.  Flow (nop 2): `.flo` as SaveFlowFile
// writes it ("PIEH", int32 w, h, w*h*2 floats; values kept as they are, so unknown ground truth stays unknown).
// Stereo (nop 1): the `.pfm` SavePFMFile writes ("Pf", w h, a negative scale; rows bottom-up, values negated).
// `what` names the file in the messages ("init-flow file").  Returns [h][w][nop] floats in `flow`, or false with a
// message in `err`.
bool read_flow_file(const char* path, int w, int h, int nop, const string& what, vector<float>& flow, string& err) {
  vector<uint8_t> b;
  if (!read_file(path, b)) {
    err = "cannot read the " + what;
    return false;
  }
  const size_t n = (size_t)w * h;
  flow.assign(n * nop, 0.f);
  if (nop == 2) {
    int32_t fw = 0, fh = 0;
    if (b.size() < 12 || memcmp(b.data(), "PIEH", 4)) {
      err = "the " + what + " is not a .flo file (PIEH)";
      return false;
    }
    memcpy(&fw, &b[4], 4);
    memcpy(&fh, &b[8], 4);
    if (fw != w || fh != h) {
      err = "the " + what + "'s size differs from the images'";
      return false;
    }
    if (b.size() != 12 + n * 2 * sizeof(float)) {
      err = "the .flo file's length does not match its header";
      return false;
    }
    memcpy(flow.data(), &b[12], n * 2 * sizeof(float));
    return true;
  }
  // three header lines: "Pf", "w h", scale
  size_t pos = 0, eol[3];
  for (int k = 0; k < 3; ++k) {
    while (pos < b.size() && pos < 256 && b[pos] != '\n') ++pos;
    if (pos >= b.size() || b[pos] != '\n') {
      err = "the " + what + " is not a .pfm file";
      return false;
    }
    eol[k] = pos++;
  }
  const string l0((const char*)&b[0], eol[0]), l1((const char*)&b[eol[0] + 1], eol[1] - eol[0] - 1),
      l2((const char*)&b[eol[1] + 1], eol[2] - eol[1] - 1);
  int fw = 0, fh = 0;
  char tail = 0;
  if (l0 != "Pf" || sscanf(l1.c_str(), "%d %d %c", &fw, &fh, &tail) != 2) {
    err = "the " + what + " is not a one-channel .pfm file (Pf)";
    return false;
  }
  char* end = nullptr;
  const double scale = strtod(l2.c_str(), &end);
  if (end == l2.c_str() || !(scale < 0)) {
    err = "the .pfm file's scale is not negative (little endian)";
    return false;
  }
  if (fw != w || fh != h) {
    err = "the " + what + "'s size differs from the images'";
    return false;
  }
  if (b.size() - pos != n * sizeof(float)) {
    err = "the .pfm file's length does not match its header";
    return false;
  }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float v;
      memcpy(&v, &b[pos + ((size_t)(h - 1 - y) * w + x) * sizeof(float)], sizeof(float));
      flow[(size_t)y * w + x] = -v;
    }
  return true;
}

// preprocess.initflow_from_fullres on the replicate-padded flow (run_dense.cpp:372-374): every value times
// 2^-(lv_f+1), then cv::resize(INTER_AREA) by s = 2^(lv_f+1) in OpenCV's area-fast order -- sum = 0, groups of four
// row-major terms add as sum += ((t0 + t1) + t2) + t3, times 1/s^2; for s = 2 with one channel ((a + b) + (c + d)) * 0.25.
ImageF initflow_level(const ImageF& padded, int lv_f) {
  const int s = 1 << (lv_f + 1);
  const float sc = ldexpf(1.f, -(lv_f + 1)), inv_area = ldexpf(1.f, -2 * (lv_f + 1));
  ImageF d;
  d.w = padded.w / s;
  d.h = padded.h / s;
  d.c = padded.c;
  d.px.resize((size_t)d.w * d.h * d.c);
  for (int y = 0; y < d.h; ++y)
    for (int x = 0; x < d.w; ++x)
      for (int k = 0; k < d.c; ++k) {
        auto t = [&](int i) { return padded.at(x * s + (i & (s - 1)), y * s + i / s, k) * sc; };
        if (s == 2 && d.c == 1) {
          d.at(x, y, k) = ((t(0) + t(1)) + (t(2) + t(3))) * 0.25f;
          continue;
        }
        float sum = 0.f;
        for (int i = 0; i < s * s; i += 4) sum += ((t(i) + t(i + 1)) + t(i + 2)) + t(i + 3);
        d.at(x, y, k) = sum * inv_area;
      }
  return d;
}

// Parameter block of the command line: nothing, one operating-point digit, or the 20 explicit
// numbers (run_dense.cpp:219-294, README.md:66-88).
struct CliParams {
  int lv_f, lv_l, maxiter, miniter, patchsz, patnorm, costfct, tv_innerit, tv_solverit, verbosity;
  float mindprate, mindrrate, minimgerr, poverl, tv_alpha, tv_gamma, tv_delta, tv_sor;
  bool usefbcon, usetvref;
};

// The four operating points (README.md:44-64 of the reference; run_dense.cpp:236-262): patch size, overlap, how many
// levels below the automatically selected coarsest one the pyramid descends, Gauss-Newton iterations (max = min),
// variational refinement on/off.  Index 0 is unused.
struct OperatingPoint { int patchsz; float poverl; int levels_down, iters; bool usetvref; };
const OperatingPoint kOperatingPoints[5] = {
    {0, 0.f, 0, 0, false}, {8, 0.3f, 2, 16, false}, {8, 0.4f, 2, 12, true}, {12, 0.75f, 4, 16, true}, {12, 0.75f, 5, 128, true}};

void parse_cli_params(int nnum, char** num, int width_org, CliParams& P) {
  // defaults shared by all operating points
  P.mindprate = 0.05f; P.mindrrate = 0.95f; P.minimgerr = 0.0f;
  P.usefbcon = false; P.patnorm = 1; P.costfct = 0;
  P.tv_alpha = 10.0f; P.tv_gamma = 10.0f; P.tv_delta = 5.0f;
  P.tv_innerit = 1; P.tv_solverit = 3; P.tv_sor = 1.6f;
  P.verbosity = 2;
  if (nnum <= 1) {
    int op = nnum == 1 ? atoi(num[0]) : 2;
    if (op < 1 || op > 4) op = 2;  // anything else selects operating point 2, like the reference's default branch
    const OperatingPoint& o = kOperatingPoints[op];
    P.patchsz = o.patchsz;
    P.poverl = o.poverl;
    P.lv_f = AutoFirstScaleSelect(width_org, 5, o.patchsz);
    P.lv_l = std::max(P.lv_f - o.levels_down, 0);
    P.maxiter = P.miniter = o.iters;
    P.usetvref = o.usetvref;
    return;
  }
  // the 20 explicit numbers, in the order of the reference's README (README.md:66-88)
  const struct { char kind; void* dst; } fields[20] = {
      {'i', &P.lv_f}, {'i', &P.lv_l}, {'i', &P.maxiter}, {'i', &P.miniter}, {'f', &P.mindprate}, {'f', &P.mindrrate},
      {'f', &P.minimgerr}, {'i', &P.patchsz}, {'f', &P.poverl}, {'b', &P.usefbcon}, {'i', &P.patnorm}, {'i', &P.costfct},
      {'b', &P.usetvref}, {'f', &P.tv_alpha}, {'f', &P.tv_gamma}, {'f', &P.tv_delta}, {'i', &P.tv_innerit},
      {'i', &P.tv_solverit}, {'f', &P.tv_sor}, {'i', &P.verbosity}};
  for (int k = 0; k < 20; ++k) {
    if (fields[k].kind == 'i') *static_cast<int*>(fields[k].dst) = atoi(num[k]);
    else if (fields[k].kind == 'f') *static_cast<float*>(fields[k].dst) = (float)atof(num[k]);
    else *static_cast<bool*>(fields[k].dst) = atoi(num[k]) != 0;
  }
}

double elapsed_ms(timeval& a) {
  timeval b;
  gettimeofday(&b, NULL);
  double tt = (b.tv_sec - a.tv_sec) * 1000.0f + (b.tv_usec - a.tv_usec) / 1000.0f;
  a = b;
  return tt;
}

}  // namespace

#ifdef OFDIS_IMGDUMP
// Test tool (no GPU): ofdis_imgdump <in.png|pgm|ppm> <gray|color> <out.pnm> -- what load_image() hands to
// the pipeline, so that tests can compare the decoders with cv2.imread (tests/test_params_io.py).
int main(int argc, char** argv) {
  if (argc != 4) return 2;
  Image8 im;
  const int want = !strcmp(argv[2], "gray") ? 1 : 3;
  if (!load_image(argv[1], want, im)) return 1;
  FILE* f = fopen(argv[3], "wb");
  if (!f) return 3;
  fprintf(f, "P%d\n%d %d\n255\n", want == 1 ? 5 : 6, im.w, im.h);
  fwrite(im.px.data(), 1, im.px.size(), f);  // colour: BGR order, as cv::imread returns it
  fclose(f);
  return 0;
}
#elif defined(OFDIS_BATCH)
// Batch front-end (SURVEY 8f rank 4): many pairs per launch through the C-ABI's frame dimension.
//
//   run_*_*_batch listfile [--batch N] [oppoint | p1 .. p20]
//
// listfile: one "image1 image2 outputfile" triple per line.  Consecutive pairs of the same size are
// grouped into batches of up to N (default 64): 8-bit frames up, pyramid / hot path / upsampling
// on the device, full-resolution flows back.  Every output is byte-identical to what the
// single-pair binary writes for that pair.
//
// Video: pair k+1 continues pair k when its image1 path is pair k's image2 path (string equality).  A batch of two
// or more pairs in which every pair continues the one before it is a clip of n+1 frames: each frame is decoded
// once and the clip goes up with ofdis_upload_sequence_u8 (each frame uploaded and its levels built once).  A
// batch that starts with the frame the previous one ended on takes that frame's decoded image over.  Every other
// batch goes through ofdis_upload_frames_u8.
//
// --warm-start (latency mode for video): pairs run one per launch, padded to multiples of 2^(lv_f+1) as a run with
// an init flow is (run_dense.cpp:301).  A pair that continues the previous one starts from that pair's flow
// (ofdis_set_initflow_from_result); the first pair of a chain starts from zero.  Each output equals what the
// single-pair binary writes given `1 <previous output>` (an all-zero flow for a chain's first pair).  Chaining makes
// a clip serial, so this mode trades throughput for the warm start.
//
// --bidirectional: every pair also runs backward (image2 -> image1; stereo: the right view's disparity, as the
// right camera), in the same launch.  A chained batch goes up with ofdis_upload_sequence_bidir_u8, any other batch
// as its pairs followed by their swapped copies (marked with ofdis_set_swapped_slots).  For an output path
// <stem><ext> it writes <stem><ext> (the forward flow, the same bytes as without the flag), <stem>_bw<ext> (the
// backward flow / right disparity) and <stem>_occ.pgm, the forward slot's consistency mask
// (ofdis_consistency_fullres with alpha 0.01, beta 0.5 for flow and 0, 1 for stereo) as binary PGM: 0 consistent,
// 255 inconsistent, 128 the flow leaves the frame.
//
// --gt gtlist: evaluation against ground truth.  gtlist holds whitespace-separated ground-truth paths, one per pair
// of the list file, in order: `.flo` for flow (unknown values kept as they are), the `.pfm` the stereo binaries write
// for stereo (this library's disparity sign).  Every file is read and checked against its pair's image size before
// any device work: a missing gtlist, an unreadable file or a wrong size exits with 1, a gtlist whose count differs
// from the list file's with 2.  After each batch the forward slots are evaluated (ofdis_flow_error_fullres; with
// --bidirectional the forward consistency mask is the class map, nclasses 3).  With verbosity > 0 these lines follow
// the TIME line:
//   EVAL (<P> pairs) n <N> epe <mean> over1 <%> over3 <%> over5 <%> outliers <%>
// and with --bidirectional one more per class, `EVAL consistent (...)`, `EVAL inconsistent (...)`, `EVAL leaves (...)`.
// The totals add the per-pair stats in list order (sum_err in float64; the all-pixel line adds a pair's classes in
// class order); epe = sum_err / n, percentages 100 * count / n, printed with %.6f; a line with n = 0 prints nan for
// every value but n.  The output files keep their bytes.  A ground-truth file that starts with the PNG signature is
// read as KITTI's 16-bit ground truth: flow RGB16, (R - 32768) / 64 and (G - 32768) / 64 where B > 0; stereo gray16,
// -(value / 256) (this library's sign) where the value is > 0; NaN (unknown) elsewhere.
//
// --kitti: every output (and with --bidirectional every _bw output) is written as KITTI's 16-bit PNG, whatever its
// extension, encoded on the device (ofdis_get_flow_fullres_encoded, OFDIS_ENC_KITTI), so 6 (flow) or 2 (stereo)
// bytes per pixel come back instead of 8 or 4.  Flow: RGB16 (u * 64 + 2^15, v * 64 + 2^15, 1), (0, 0, 0) where the
// flow is NaN; stereo: gray16 d * 256 of the positive disparity d (the left view's -F, a _bw file's right-view +F),
// clamped to [1, 65535], 0 where d is negative or NaN.  The _occ.pgm masks and the EVAL lines do not change.
//
// --color: every output also gets <stem>_color.png (with --bidirectional also <stem>_bw_color.png), an 8-bit RGB PNG
// of the flow colored on the device (ofdis_flow_color_fullres): Middlebury's color wheel for flow, the color map of
// KITTI's stereo devkit for the positive disparity (a _bw file's right-view +F).  Each pair is colored with its own
// maximum, as Middlebury's tool does; --color-max M (a positive finite number; it needs --color) colors every pair
// with the scale M, so that the frames of a clip compare.  3 bytes per pixel come back for it.  The other output files
// keep their bytes.
//
// --confidence R (1 <= R <= 7): every pair also gets <stem>_conf.pfm, the forward slot's per-pixel confidence
// (ofdis_confidence_fullres with radius R, s_fb 1, s_tex 100 and min_count (2R+1)^2 / 2, integer division) as float32
// in [0, 1], stored as is (read_pfm returns it negated, as it returns every PFM of this front-end).  The forward-backward
// term is used when the backward slots already run (--bidirectional, --lr-check, --interpolate or --tracks); no flag
// adds them.  With verbosity > 0 every batch prints `CONF pairs N mean M`, M the float64 mean over the batch's pixels
// (%.9g).  Not with --warm-start; every other output keeps its bytes.
//
// --interpolate T (0 < T < 1): every pair also gets <stem>_interp.png, the frame at time T between image1 and image2
// synthesised on the device from the pair's forward and backward flows (ofdis_interpolate_fullres, with the
// consistency thresholds of --bidirectional): 8-bit gray from the *_INT binaries, 8-bit RGB from the *_RGB binaries
// (computed on the decoder's BGR order, written as RGB).  The backward slots run in the same launch, as with
// --bidirectional, but the _bw and _occ files are only written when --bidirectional is given too; every other output
// keeps its bytes.  Not with --warm-start.
//
// --tracks PATH: dense point trajectories through the pairs (ofdis_track_begin / ofdis_track_advance).  A pair that
// does not continue the previous one starts a new clip with ofdis_track_begin on its image1; the pairs of a clip
// continue the same tracker, across batches.  Settings: spacing 8, capacity 4 x the cells, alpha/beta of
// --bidirectional, mb_alpha 0.01, mb_beta 0.002 (Sundaram et al.'s motion-boundary test), min_eig 25 (about 1 grey
// level^2 per pixel over the 5 x 5 window).  PATH gets the header `# clip frame id x y`, then one line per live track
// and frame, clips and frames counted from 0, x and y printed with %.9g (which round-trips float32).  The backward
// slots run in the same launch, as with --interpolate; every other output keeps its bytes.  With verbosity > 0 a
// line `TRACKS clips C frames N seeded S leaves L inconsistent I boundary B dropped D` follows the TIME line.  Not
// with --warm-start.
//
// Stereo binaries only (the flow binaries refuse these flags, and so does --warm-start): filtered disparities
// (ofdis_disparity_fullres) of every pair's left view.  --lr-check invalidates the pixels that fail the left-right
// check of --bidirectional (alpha 0, beta 1; the backward slots run in the same launch, the _bw and _occ files are only
// written when --bidirectional is given too); --speckle N R removes the components of at most N pixels whose
// 4-neighbours differ by at most R px; --fill fills the holes with the background disparity; --camera
// fx,fy,cx,cy,baseline,doffs gives depth and points.  With any of them every pair also gets <stem>_filtered<ext>, the
// filtered disparity in the format and sign of <stem><ext> (PFM of the positive disparity, NaN where invalid; with
// --kitti KITTI's 16-bit PNG with NaN as 0).  With --camera also <stem>_depth.pfm (Z as is, NaN where invalid) and
// <stem>.ply, a binary little-endian point cloud of the pixels with a finite Z in row-major order: float x, y, z, then
// uchar red, green, blue from image1 (gray replicated).  With verbosity > 0 every batch prints a line
// `DISP pairs N valid V inconsistent I leaves L range R speckle S filled F` (the status counts, and the pixels of
// another status that got a value).  Every other output keeps its bytes.
//
// --global-motion MODEL PATH (flow binaries only; MODEL similarity, affine or homography): the camera motion of every
// pair (ofdis_global_motion_fullres) with step 8, 1024 hypotheses, a 1 px threshold, 3 refits and seed 0; with
// --bidirectional only the correspondences whose consistency mask of --bidirectional (alpha 0.01, beta 0.5) is 0.
// PATH gets one line per pair, `stem m00 m01 m02 m10 m11 m12 m20 m21 m22 status n_corr n_inliers`, stem the output
// path without its extension and the model (mapping an image1 pixel to its image2 position) printed with %.17g
// (which round-trips float64).  Every pair also gets <stem>_residual<ext>, the flow minus the model's flow, in the
// format of <stem><ext> (KITTI's 16-bit PNG with --kitti); <stem>_moving.pgm, 0 where a pixel moves with the camera,
// 255 where it moves on its own and 128 where its flow is unknown, leaves the frame or (with --bidirectional) is
// inconsistent, the code of _occ.pgm; and <stem>_registered.png, image2 sampled at the model's position of every
// pixel of image1 (0 outside image2).  Every other output keeps its bytes.  Not with --warm-start.
//
// --descriptors PATH (needs --tracks, whose clips it describes; flow binaries only): the trajectory descriptors of
// every clip's tracks (ofdis_traj_begin / ofdis_traj_advance in place of the tracker's calls, whose tracks they keep
// bit for bit), with the --global-motion models when that flag is given and without camera compensation otherwise.
// Settings: Wang and Schmid's, L 15, nt 3, N 32, ns 2, min_flow 0.4, eps 0.05, min_disp 1, min_var sqrt(3), max_var 50,
// max_dis 20.  PATH gets the header `# clip id start mean_x mean_y sd_x sd_y length d0 .. d425`, then one line per
// emitted segment in the order of the calls, clips counted from 0 and start from the clip's first frame, every float
// printed with %.9g (which round-trips float32).  With verbosity > 0 a line `DESCRIPTORS clips C emitted E static S
// erratic R jump J camera K` follows the TRACKS line.  Frames smaller than N are refused before any device work; every
// other output, the --tracks file included, keeps its bytes.  Not with --warm-start.
//
// --fisher CODEBOOK PATH (needs --tracks; flow binaries only): one improved Fisher vector per clip of --tracks from the
// descriptors of --descriptors' stage (run whether or not --descriptors is given), encoded on the device with the
// codebook file CODEBOOK (preprocess.write_fisher_codebook's format, whose desc_dim and block ranges must be the
// descriptors': 426 floats, blocks 0+30, 30+96, 126+108, 234+96, 330+96).  Without --descriptors the descriptors go
// from the descriptor stage to the encoder on the device (ofdis_traj_advance_fisher); with it they are pushed from the
// host copy that --descriptors writes.  PATH gets the header `# clip n_desc n_0 .. n_{B-1} fv0 .. fv{F-1}`, then at
// every clip's end one line: the clip, the descriptors pushed, each block's N_b and the vector's F floats with %.9g.
// With verbosity > 0 a line `FISHER clips C descriptors N skipped s_0 .. s_{B-1}` follows the DESCRIPTORS line.  The
// stereo binaries, --warm-start, a missing --tracks, an unreadable, malformed or mismatched codebook and an unwritable
// PATH are refused before any device work; every other output keeps its bytes.
//
// --stabilize RADIUS CROP DIR (needs --global-motion, whose models it smooths; flow binaries only): every clip
// stabilised on the device (ofdis_stab_begin / ofdis_stab_push / ofdis_stab_finish).  Clips are the runs of pairs of
// --tracks, across batches: the stabiliser begins on a clip's first image1, every batch pushes the image2 frames of
// its run with their models and the clip's end emits the rest.  Settings: radius RADIUS (1 .. 64), Gaussian weights
// exp(-d*d / (2 RADIUS)) (sigma^2 = RADIUS, OpenCV videostab's default), crop CROP (0 <= CROP < 0.5) with the limit on
// when CROP > 0.  Every frame of every clip goes to DIR/stab_<clip %04d>_<frame %06d>.png (8-bit gray, or RGB from the
// *_RGB binaries), clips and frames counted from 0, and DIR/stab.txt gets one line per frame,
// `clip frame s00 s01 s02 s10 s11 s12 s20 s21 s22 lambda status`, the correction and its share printed with %.17g.
// Every other output keeps its bytes.  Not with --warm-start.

// --scene-flow DISPLIST (flow binaries only): scene flow (ofdis_scene_flow_fullres, edge_diff 1) of every pair from
// its forward flow and two disparity maps.  DISPLIST holds two files per pair, in list order: the disparity of image1
// and that of image2, each a PFM of the positive disparity (what run_DE_*_batch writes, <stem>_filtered.pfm included;
// NaN unknown) or KITTI's 16-bit disparity PNG (0 unknown).  Every pair gets <stem>_disp1.pfm, image2's disparity
// warped to image1 (PFM of the positive disparity, NaN unknown); with --kitti <stem>_disp1<ext>, KITTI's 16-bit
// disparity PNG (NaN as 0), so that <stem><ext>, the disparity of image1 and this file form a KITTI scene-flow
// submission.  With --camera fx,fy,cx,cy,baseline,doffs also <stem>_sceneflow.pfm, a 3-channel PFM ("PF", rows
// bottom-up) of the 3-D motion, NaN where unknown.  --gt-scene-flow GTLIST holds three files per pair: the ground-truth
// disparities at t and at t+1 (KITTI's disp_occ_0 and disp_occ_1, PFM or PNG as above) and the flow (KITTI PNG or
// .flo).  With verbosity > 0 every pair prints `SFEVAL <out> d1 O N P d2 O N P fl O N P sf O N P` (outliers, pixels
// counted, percentage; KITTI's D1, D2, Fl and SF with an unknown estimate counted as an outlier) and the end
// `SFEVAL (<P> pairs) ...`, with --bidirectional also per class of the forward consistency mask as EVAL.  A list
// whose count or files do not match the pairs is refused before any device work; every other output keeps its
// bytes.  Not with --warm-start; --camera on a flow binary needs --scene-flow.

// --odometry DIR (flow binaries only, with --scene-flow and --camera, which give both disparities of every pair and the
// stereo camera): the rig's ego-motion of every pair (ofdis_egomotion_fullres) with step 8, 1024 hypotheses, a 1 px
// threshold, 5 Gauss-Newton rounds, seed 0 and edge_diff 1; with --bidirectional only correspondences whose forward
// consistency mask (the thresholds of _occ.pgm) is 0.  A clip is a run of pairs whose image1 is the previous pair's
// image2; clips and their frames count from 0.  DIR/odometry.txt gets one line per pair, `clip frame status n_corr
// ransac_inliers n_inliers` and the 12 numbers of the relative pose [R | t] (camera t to camera t+1, row-major, %.17g);
// DIR/poses_<clip %04d>.txt the clip's camera-to-world poses in KITTI's odometry format, n+1 lines from the identity,
// T_(k+1) = T_k inv([R | t]_k).  Every pair gets <stem>_objects.pgm (0 static, 255 moves on its own, 128 unknown: the
// code of _occ.pgm) and <stem>_objmotion.pfm (3-channel PFM as _sceneflow.pfm, the object's own 3-D motion, NaN where
// unknown).  --gt-poses LIST holds one KITTI poses file per clip, with at least n+1 lines for a clip of n pairs; with
// verbosity > 0 every pair prints `ODOEVAL clip frame t_err r_err` (the relative pose error in metres and degrees, as
// KITTI's devkit forms it) and the end `ODOEVAL (<P> pairs) t_err <mean> r_err <mean>`.  Refused before any device
// work: the stereo binaries, --warm-start, --odometry without --scene-flow or --camera, --gt-poses without
// --odometry, a list that does not match the clips or a file with too few lines, and a DIR that cannot be written.
// Every other output keeps its bytes.
//
// --mono-odometry DIR with --intrinsics fx,fy,cx,cy (flow binaries only): the monocular relative pose of every pair
// (ofdis_relpose_fullres) with step 8, 1024 hypotheses, a 1 px Sampson threshold, 5 Gauss-Newton rounds, a 0.5 px
// parallax guard and seed 0; with --bidirectional only correspondences whose forward consistency mask is 0.
// DIR/monodometry.txt gets one line per pair, `clip frame status` and the 12 numbers of [R | t] with |t| = 1 (camera
// t to camera t+1, row-major, %.17g, NaN unless status 0); DIR/poses_<clip %04d>.txt the clip's camera-to-world poses
// as --odometry writes them, chained with unit steps, or with --gt-poses with the ground truth's step lengths.  Every
// pair gets <stem>_epimask.pgm (0 epipolar inlier, 255 outlier, 128 unknown) and <stem>_depthrel.pfm (1-channel PFM,
// the depth at image1 in units of the step, NaN where unknown).  With --gt-poses and verbosity > 0 every pair prints
// `MONOEVAL clip frame r_err t_dir_err` (degrees) and the end `MONOEVAL (<P> pairs) r_err <mean> t_dir_err <mean>`
// over the pairs of status 0.  Refused before any device work: the stereo binaries, --warm-start, --mono-odometry
// without --intrinsics or the reverse, intrinsics that are not four finite numbers with fx, fy > 0, and a DIR that
// cannot be written.  --gt-poses is valid with --odometry or --mono-odometry; with both, the two share its poses
// files and --mono-odometry's poses files are DIR/poses_<clip>.txt of its own DIR.
//
// --fuse voxel,trunc,x0,y0,z0,nx,ny,nz (needs --odometry, whose poses place the disparities): one TSDF volume per clip
// of --odometry (ofdis_fuse_begin / ofdis_fuse_push / ofdis_fuse_extract), nx x ny x nz voxels of `voxel` metres from
// (x0, y0, z0) in the clip's first camera, truncation `trunc` metres, max_weight 64, max_depth +inf, with colour.  The
// clip's first pair begins it; every pair pushes its image1 disparity (the first map of its DISPLIST line) with its
// chained pose T_k of DIR/poses_<clip>.txt and image1's colours, and the clip's last pair also pushes image2's
// disparity with T_n and image2's colours.  At the clip's end the zero crossings of weight >= 1 go to
// DIR/fused_<clip %04d>.ply, a binary little-endian PLY of float x, y, z, nx, ny, nz and uchar red, green, blue, in
// the volume's order (preprocess.fuse_extract, preprocess.write_fused_ply).  With verbosity > 0 every clip prints
// `FUSE clip C frames F points P`.  Refused before any device work: --fuse without --odometry, the stereo binaries,
// --warm-start and a spec that is not 8 numbers with voxel and trunc > 0, sizes >= 1 and at most 2^30 voxels.  Every
// other output keeps its bytes.
//
// --mesh (with --fuse): at each clip's end also DIR/fused_<clip %04d>_mesh.ply, the same volume's triangle mesh of
// weight >= 1 (ofdis_fuse_mesh): the vertices of fused_<clip>.ply, then `element face F` with `property list uchar uint
// vertex_indices` (preprocess.fuse_mesh, preprocess.write_fused_mesh_ply).  With verbosity > 0 every clip prints
// `MESH clip C vertices V faces F`.  Refused before any device work: --mesh without --fuse, and whatever --fuse
// refuses.  Every other output keeps its bytes.

// The fused points (with mesh, the mesh) as a binary little-endian PLY: float x, y, z, nx, ny, nz and uchar red,
// green, blue per vertex, then with mesh nf faces of uchar 3 and three uint vertex indices.  False when it cannot be
// written.
static bool write_fused_ply(const string& path, const ofdis_fuse_point* pts, long count, int nochannels, bool mesh,
                            const unsigned int* faces, long nf) {
  FILE* pf = fopen(path.c_str(), "wb");
  if (!pf) return false;
  fprintf(pf, "ply\nformat binary_little_endian 1.0\nelement vertex %ld\nproperty float x\nproperty float y\n"
              "property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
              "property uchar green\nproperty uchar blue\n", count);
  if (mesh) fprintf(pf, "element face %ld\nproperty list uchar uint vertex_indices\n", nf);
  fprintf(pf, "end_header\n");
  vector<uint8_t> buf((size_t)27 * count + (mesh ? (size_t)13 * nf : 0));
  for (long i = 0; i < count; ++i) {
    const ofdis_fuse_point& q = pts[i];
    memcpy(&buf[(size_t)27 * i], &q.x, 24);
    // the decoder's BGR: channel 2 is red (gray: all three equal)
    const uint8_t rgb[3] = {nochannels == 3 ? q.b : q.r, q.g, nochannels == 3 ? q.r : q.b};
    memcpy(&buf[(size_t)27 * i + 24], rgb, 3);
  }
  for (long i = 0; mesh && i < nf; ++i) {
    uint8_t* f = &buf[(size_t)27 * count + (size_t)13 * i];
    f[0] = 3;
    memcpy(f + 1, faces + (size_t)3 * i, 12);
  }
  bool wrote = fwrite(buf.data(), 1, buf.size(), pf) == buf.size();
  return fclose(pf) == 0 && wrote;
}

// Rigid poses as 12 doubles, row-major [R | t].  T <- T inv(P): the next camera-to-world pose of a clip (KITTI's
// odometry convention) from the relative pose P, camera t to camera t+1.
static void chain_pose(double* T, const double* P) {
  double I[12];  // inv(P) = [R^T | -R^T t]
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) I[4 * i + j] = P[4 * j + i];
    I[4 * i + 3] = -(P[i] * P[3] + P[4 + i] * P[7] + P[8 + i] * P[11]);
  }
  double N[12];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j)
      N[4 * i + j] = T[4 * i] * I[j] + T[4 * i + 1] * I[4 + j] + T[4 * i + 2] * I[8 + j] + (j == 3 ? T[4 * i + 3] : 0.0);
  memcpy(T, N, sizeof(N));
}

// The relative pose error of the estimate P (camera t to t+1) against the ground-truth camera-to-world poses G0, G1,
// as KITTI's devkit forms it: E = inv(inv(G0) G1) inv(P), t_err = |E_t| (metres), r_err = acos((trace(E_R) - 1) / 2)
// in degrees.
static void pose_error(const double* G0, const double* G1, const double* P, double* t_err, double* r_err) {
  // inv(inv(G0) G1) = inv(G1) G0; then E = inv(G1) G0 inv(P): chain G0 by P gives G0 inv(P)
  double A[12], Gi[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  memcpy(A, G0, sizeof(A));
  chain_pose(A, P);   // A = G0 inv(P)
  chain_pose(Gi, G1);  // Gi = inv(G1)
  double E[12];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j)
      E[4 * i + j] = Gi[4 * i] * A[j] + Gi[4 * i + 1] * A[4 + j] + Gi[4 * i + 2] * A[8 + j] + (j == 3 ? Gi[4 * i + 3] : 0.0);
  *t_err = sqrt(E[3] * E[3] + E[7] * E[7] + E[11] * E[11]);
  const double c = 0.5 * (E[0] + E[5] + E[10] - 1.0);
  *r_err = acos(fmin(1.0, fmax(-1.0, c))) * (180.0 / M_PI);
}

// <stem><ext> -> <stem><suffix><ext> (ext: from the last '.' of the file name, empty if it has none)
static string with_suffix(const string& path, const char* suffix, const char* new_ext = nullptr) {
  const size_t slash = path.find_last_of('/'), dot = path.find_last_of('.');
  const size_t cut = (dot != string::npos && (slash == string::npos || dot > slash)) ? dot : path.size();
  return path.substr(0, cut) + suffix + (new_ext ? string(new_ext) : path.substr(cut));
}

// width and height from an image file's header (binary PNM, or PNG's IHDR, which the format puts first)
static bool image_size(const char* path, int& w, int& h) {
  vector<uint8_t> b, rgb;
  if (!read_file(path, b)) return false;
  Image8 im;
  int ch = 0;
  if (decode_pnm(b, im, rgb, ch)) {
    w = im.w;
    h = im.h;
    return true;
  }
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (b.size() < 24 || memcmp(b.data(), sig, 8) || memcmp(&b[12], "IHDR", 4)) return false;
  w = (int)be32(&b[16]);
  h = (int)be32(&b[20]);
  return w > 0 && h > 0;
}

// one EVAL line: `label` is empty for all pixels, else the class name
static void print_eval(const char* label, size_t pairs, const ofdis_error_stats& s) {
  printf("EVAL %s%s(%zu pairs) n %lld", label, *label ? " " : "", pairs, s.n);
  if (s.n == 0) {
    printf(" epe nan over1 nan over3 nan over5 nan outliers nan\n");
    return;
  }
  const double n = (double)s.n;
  printf(" epe %.6f over1 %.6f over3 %.6f over5 %.6f outliers %.6f\n", s.sum_err / n, 100.0 * (double)s.n_over[0] / n,
         100.0 * (double)s.n_over[1] / n, 100.0 * (double)s.n_over[2] / n, 100.0 * (double)s.n_outlier / n);
}

static void add_stats(ofdis_error_stats& t, const ofdis_error_stats& s) {
  t.n += s.n;
  for (int k = 0; k < 3; ++k) t.n_over[k] += s.n_over[k];
  t.n_outlier += s.n_outlier;
  t.sum_err += s.sum_err;
}

static void add_sf_stats(ofdis_sf_stats& t, const ofdis_sf_stats& s) {
  t.n_d1 += s.n_d1; t.n_d2 += s.n_d2; t.n_fl += s.n_fl; t.n_sf += s.n_sf;
  t.out_d1 += s.out_d1; t.out_d2 += s.out_d2; t.out_fl += s.out_fl; t.out_sf += s.out_sf;
}

// one SFEVAL line: a pair's output path (pairs 0), or the total of `pairs` pairs with the class name (empty: all)
static void print_sfeval(const char* label, size_t pairs, const ofdis_sf_stats& s) {
  if (pairs) printf("SFEVAL %s%s(%zu pairs)", label, *label ? " " : "", pairs);
  else printf("SFEVAL %s", label);
  const long long n[4] = {s.n_d1, s.n_d2, s.n_fl, s.n_sf}, o[4] = {s.out_d1, s.out_d2, s.out_fl, s.out_sf};
  static const char* const kNames[4] = {"d1", "d2", "fl", "sf"};
  for (int i = 0; i < 4; ++i) {
    if (n[i]) printf(" %s %lld %lld %.6f", kNames[i], o[i], n[i], 100.0 * (double)o[i] / (double)n[i]);
    else printf(" %s %lld %lld nan", kNames[i], o[i], n[i]);
  }
  printf("\n");
}

// a 3-channel PFM ("PF", w h, scale -1: little endian, rows bottom-up) of [h][w][3] floats, written as they are
static void save_pfm3(const float* v, int w, int h, const char* filename) {
  FILE* f = fopen(filename, "wb");
  if (!f) {
    cout << "WriteFile: could not open file" << endl;
    return;
  }
  fprintf(f, "PF\n%d %d\n%f\n", w, h, -1.0f);
  for (int y = h - 1; y >= 0; --y)
    if (fwrite(v + (size_t)y * w * 3, sizeof(float), (size_t)w * 3, f) != (size_t)w * 3)
      cout << "WriteFile: problem writing data" << endl;
  fclose(f);
}

static const uint8_t kPngSig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};

// KITTI ground truth: a 16-bit non-interlaced PNG of the image size, RGB16 for flow (nop 2), gray16 for stereo, every
// row filter 0-4 undone with a byte distance of 2 * channels.  Returns [h][w][nop] floats in this library's
// convention with NaN for the invalid pixels (kitti_to_flow of of_dis_b200/preprocess.py), or false with `err`.
static bool read_kitti_png(const vector<uint8_t>& b, int w, int h, int nop, const string& what, vector<float>& flow,
                           string& err) {
  size_t pos = 8;
  int iw = 0, ih = 0, depth = 0, ctype = -1, interlace = -1;
  vector<uint8_t> idat;
  while (pos + 12 <= b.size()) {
    const uint32_t len = be32(&b[pos]);
    const char* type = (const char*)&b[pos + 4];
    const uint8_t* data = &b[pos + 8];
    if (len > b.size() - pos - 12) break;
    if (!memcmp(type, "IHDR", 4) && len >= 13) {
      iw = (int)be32(data);
      ih = (int)be32(data + 4);
      depth = data[8];
      ctype = data[9];
      interlace = data[12];
    } else if (!memcmp(type, "IDAT", 4)) idat.insert(idat.end(), data, data + len);
    else if (!memcmp(type, "IEND", 4)) break;
    pos += 12 + len;
  }
  const int ch = nop == 2 ? 3 : 1;
  if (depth != 16 || ctype != (nop == 2 ? 2 : 0) || interlace != 0) {
    err = "the " + what + " is not a 16-bit non-interlaced KITTI PNG (" + (nop == 2 ? "RGB16 flow)" : "gray16 disparity)");
    return false;
  }
  if (iw != w || ih != h) {
    err = "the " + what + "'s size differs from the images'";
    return false;
  }
  const size_t stride = (size_t)w * ch * 2, bpp = 2 * ch;
  vector<uint8_t> raw((stride + 1) * h);
  uLongf rawlen = raw.size();
  if (uncompress(raw.data(), &rawlen, idat.data(), idat.size()) != Z_OK || rawlen != raw.size()) {
    err = "the " + what + "'s image data does not decompress to its size";
    return false;
  }
  vector<uint8_t> img(stride * h), zero(stride, 0);
  for (int y = 0; y < h; ++y) {
    const uint8_t ft = raw[(stride + 1) * y];
    const uint8_t* in = &raw[(stride + 1) * y + 1];
    uint8_t* out = &img[stride * y];
    const uint8_t* up = y ? &img[stride * (y - 1)] : zero.data();
    for (size_t x = 0; x < stride; ++x) {
      const int a = x >= bpp ? out[x - bpp] : 0, bb = up[x], c = x >= bpp ? up[x - bpp] : 0;
      int pr = 0;
      switch (ft) {
        case 0: pr = 0; break;
        case 1: pr = a; break;
        case 2: pr = bb; break;
        case 3: pr = (a + bb) >> 1; break;
        case 4: {
          const int p = a + bb - c, pa = abs(p - a), pb = abs(p - bb), pc = abs(p - c);
          pr = (pa <= pb && pa <= pc) ? a : (pb <= pc ? bb : c);
          break;
        }
        default:
          err = "the " + what + " has an unknown PNG row filter";
          return false;
      }
      out[x] = (uint8_t)(in[x] + pr);
    }
  }
  const float nan = std::numeric_limits<float>::quiet_NaN();
  flow.assign((size_t)w * h * nop, 0.f);
  for (size_t i = 0; i < (size_t)w * h; ++i) {
    const uint8_t* s = &img[i * bpp];
    auto sample = [s](int k) { return (float)(((unsigned)s[2 * k] << 8) | s[2 * k + 1]); };
    if (nop == 2) {
      const bool valid = sample(2) > 0.0f;
      flow[2 * i] = valid ? (sample(0) - 32768.0f) / 64.0f : nan;
      flow[2 * i + 1] = valid ? (sample(1) - 32768.0f) / 64.0f : nan;
    } else {
      flow[i] = sample(0) > 0.0f ? -(sample(0) / 256.0f) : nan;
    }
  }
  return true;
}

// a ground-truth file of --gt: KITTI's 16-bit PNG when it starts with the PNG signature, else read_flow_file's formats
static bool read_gt_file(const char* path, int w, int h, int nop, vector<float>& flow, string& err) {
  const string what = "ground-truth file";
  vector<uint8_t> b;
  if (read_file(path, b) && b.size() >= 8 && !memcmp(b.data(), kPngSig, 8)) {
    try {
      return read_kitti_png(b, w, h, nop, what, flow, err);
    } catch (const std::exception&) {  // bad_alloc / length errors on malformed headers
      err = "the " + what + " is not a readable KITTI PNG";
      return false;
    }
  }
  return read_flow_file(path, w, h, nop, what, flow, err);
}

// A PNG of one slot with `depth` 16 (uint16 samples in host order; KITTI's flow RGB16 for `ch` = 3, disparity gray16
// for 1) or 8 (bytes; the RGB color images of --color): IHDR, one IDAT of filter-0 rows with the samples big-endian,
// IEND
static void save_png(const void* samples, int w, int h, int ch, int depth, const char* filename) {
  const int bytes = depth / 8;
  const size_t stride = (size_t)w * ch * bytes;
  vector<uint8_t> raw((stride + 1) * h);
  for (int y = 0; y < h; ++y) {
    uint8_t* r = &raw[(stride + 1) * y];
    r[0] = 0;
    if (bytes == 1) {
      memcpy(r + 1, static_cast<const uint8_t*>(samples) + (size_t)y * stride, stride);
      continue;
    }
    const uint16_t* s = static_cast<const uint16_t*>(samples) + (size_t)y * w * ch;
    for (size_t k = 0; k < (size_t)w * ch; ++k) {
      r[1 + 2 * k] = (uint8_t)(s[k] >> 8);
      r[2 + 2 * k] = (uint8_t)(s[k] & 0xff);
    }
  }
  vector<uint8_t> z(compressBound(raw.size()));
  uLongf zlen = z.size();
  if (compress2(z.data(), &zlen, raw.data(), raw.size(), 1) != Z_OK) {
    cout << "WriteFile: problem compressing data" << endl;
    return;
  }
  FILE* f = fopen(filename, "wb");
  if (!f) {
    cout << "WriteFile: could not open file" << endl;
    return;
  }
  bool ok = fwrite(kPngSig, 1, 8, f) == 8;
  auto chunk = [&](const char* type, const uint8_t* data, uint32_t len) {
    uint8_t be[4] = {(uint8_t)(len >> 24), (uint8_t)(len >> 16), (uint8_t)(len >> 8), (uint8_t)len};
    uLong crc = crc32(0L, (const Bytef*)type, 4);
    if (len) crc = crc32(crc, data, len);
    const uint8_t cb[4] = {(uint8_t)(crc >> 24), (uint8_t)(crc >> 16), (uint8_t)(crc >> 8), (uint8_t)crc};
    ok = ok && fwrite(be, 1, 4, f) == 4 && fwrite(type, 1, 4, f) == 4 && (!len || fwrite(data, 1, len, f) == len) &&
         fwrite(cb, 1, 4, f) == 4;
  };
  const uint8_t ihdr[13] = {(uint8_t)(w >> 24), (uint8_t)(w >> 16), (uint8_t)(w >> 8), (uint8_t)w,
                            (uint8_t)(h >> 24), (uint8_t)(h >> 16), (uint8_t)(h >> 8), (uint8_t)h,
                            (uint8_t)depth, (uint8_t)(ch == 3 ? 2 : 0), 0, 0, 0};
  chunk("IHDR", ihdr, 13);
  chunk("IDAT", z.data(), (uint32_t)zlen);
  chunk("IEND", nullptr, 0);
  if (!ok) cout << "WriteFile: problem writing data" << endl;
  fclose(f);
}

static void save_mask_pgm(const uint8_t* mask, int w, int h, const char* filename) {
  FILE* f = fopen(filename, "wb");
  if (!f) {
    cout << "WriteFile: could not open file" << endl;
    return;
  }
  static const uint8_t level[3] = {0, 255, 128};
  vector<uint8_t> px((size_t)w * h);
  for (size_t i = 0; i < px.size(); ++i) px[i] = level[mask[i] < 3 ? mask[i] : 1];
  fprintf(f, "P5\n%d %d\n255\n", w, h);
  if (fwrite(px.data(), 1, px.size(), f) != px.size()) cout << "WriteFile: problem writing data" << endl;
  fclose(f);
}

// --fisher: a codebook file of preprocess.write_fisher_codebook ("OFDISFV1", int32 K, nblocks, desc_dim,
// offset/dim_in/dim per block, the float32 body), checked as ofdis_fisher_begin checks it
struct FisherBook {
  ofdis_fisher_codebook cb;
  vector<float> body;
};
static bool read_fisher_book(const char* path, FisherBook& fb, string& err) {
  FILE* f = fopen(path, "rb");
  if (!f) {
    err = "cannot read the codebook";
    return false;
  }
  vector<unsigned char> raw;
  unsigned char buf[65536];
  for (size_t got; (got = fread(buf, 1, sizeof(buf), f)) > 0;) raw.insert(raw.end(), buf, buf + got);
  fclose(f);
  auto i32 = [&raw](size_t at) {
    int32_t v;
    memcpy(&v, raw.data() + at, 4);
    return (int)v;
  };
  if (raw.size() < 20 || memcmp(raw.data(), "OFDISFV1", 8) != 0) {
    err = "not a codebook file (OFDISFV1)";
    return false;
  }
  memset(&fb.cb, 0, sizeof(fb.cb));
  fb.cb.K = i32(8);
  fb.cb.nblocks = i32(12);
  fb.cb.desc_dim = i32(16);
  if (fb.cb.K < 1 || fb.cb.K > 256 || fb.cb.nblocks < 1 || fb.cb.nblocks > OFDIS_FISHER_MAX_BLOCKS ||
      fb.cb.desc_dim < 1 || raw.size() < 20 + 12 * (size_t)fb.cb.nblocks) {
    err = "bad codebook header";
    return false;
  }
  const size_t K = fb.cb.K;
  size_t body = 0;
  for (int b = 0; b < fb.cb.nblocks; ++b) {
    ofdis_fisher_block& bl = fb.cb.blocks[b];
    bl.offset = i32(20 + 12 * b);
    bl.dim_in = i32(24 + 12 * b);
    bl.dim = i32(28 + 12 * b);
    if (bl.dim < 1 || bl.dim > bl.dim_in || bl.dim_in > 512 || bl.offset < 0 ||
        (long long)bl.offset + bl.dim_in > fb.cb.desc_dim) {
      err = "bad codebook block";
      return false;
    }
    body += bl.dim_in + (size_t)bl.dim * bl.dim_in + 2 * K * bl.dim + 2 * K;
  }
  const size_t at = 20 + 12 * (size_t)fb.cb.nblocks;
  if (raw.size() != at + 4 * body) {
    err = "codebook body does not match its header";
    return false;
  }
  fb.body.resize(body);
  memcpy(fb.body.data(), raw.data() + at, 4 * body);
  const float* a = fb.body.data();
  for (int b = 0; b < fb.cb.nblocks; ++b) {
    const size_t D = fb.cb.blocks[b].dim_in, P = fb.cb.blocks[b].dim;
    const size_t n[4] = {D + P * D + K * P, K * P, K, K};  // finite; isig > 0; c finite; w > 0
    for (int part = 0; part < 4; ++part)
      for (size_t i = 0; i < n[part]; ++i, ++a)
        if (!(std::fabs(*a) <= FLT_MAX) || (part % 2 == 1 && !(*a > 0.f))) {
          err = "codebook entries must be finite, isig and w > 0";
          return false;
        }
  }
  fb.cb.params = fb.body.data();
  return true;
}

// One refusal line on stderr, "error: " and the formatted message; returns `code`, the exit code.
static __attribute__((format(printf, 2, 3))) int refuse(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  fputs("error: ", stderr);
  vfprintf(stderr, fmt, ap);
  fputc('\n', stderr);
  va_end(ap);
  return code;
}

// A whitespace-separated list file (the list file, --gt, --scene-flow, --gt-scene-flow, --gt-poses): its words
static bool read_words(const char* path, vector<string>& words) {
  FILE* f = fopen(path, "r");
  if (!f) return false;
  char g[4096];
  while (fscanf(f, "%4095s", g) == 1) words.push_back(g);
  fclose(f);
  return true;
}

// The decoder's BGR order as RGB: `im` itself for gray, else `buf` holding the converted copy
static const uint8_t* as_rgb(const uint8_t* im, size_t hwc, int nochannels, vector<uint8_t>& buf) {
  if (nochannels != 3) return im;
  buf.resize(hwc);
  for (size_t q = 0; q < hwc; q += 3) {
    buf[q] = im[q + 2];
    buf[q + 1] = im[q + 1];
    buf[q + 2] = im[q];
  }
  return buf.data();
}

// KITTI's 16-bit disparity PNG of positive disparities: d * 256 clamped to [1, 65535], 0 where d is negative or NaN
static void save_kitti_disp(const float* d, int w, int h, const string& path) {
  vector<uint16_t> enc((size_t)w * h);
  for (size_t i = 0; i < enc.size(); ++i)  // NaN fails d >= 0 and is written as 0
    enc[i] = d[i] >= 0.0f ? (uint16_t)fminf(fmaxf(d[i] * 256.0f, 1.0f), 65535.0f) : (uint16_t)0;
  save_png(enc.data(), w, h, 1, 16, path.c_str());
}

// KITTI's 16-bit flow PNG, the encoding of OFDIS_ENC_KITTI: (u * 64 + 2^15, v * 64 + 2^15, 1), (0, 0, 0) where NaN
static void save_kitti_flow(const float* f, int w, int h, const string& path) {
  vector<uint16_t> enc((size_t)3 * w * h);
  for (size_t i = 0; i < (size_t)w * h; ++i) {
    const float u = f[2 * i], v = f[2 * i + 1];
    const bool valid = !std::isnan(u) && !std::isnan(v);
    enc[3 * i] = valid ? (uint16_t)fminf(fmaxf(u * 64.0f + 32768.0f, 0.0f), 65535.0f) : (uint16_t)0;
    enc[3 * i + 1] = valid ? (uint16_t)fminf(fmaxf(v * 64.0f + 32768.0f, 0.0f), 65535.0f) : (uint16_t)0;
    enc[3 * i + 2] = valid ? 1 : 0;
  }
  save_png(enc.data(), w, h, 3, 16, path.c_str());
}

// A 1-channel PFM holding v as it is (a positive disparity, a depth): SavePFMFile writes -value, so v goes in negated
static void save_pfm1(const float* v, int w, int h, const string& path) {
  ImageF f;
  f.w = w;
  f.h = h;
  f.c = 1;
  f.px.resize((size_t)w * h);
  for (size_t i = 0; i < f.px.size(); ++i) f.px[i] = -v[i];
  SavePFMFile(f, path.c_str());
}

// Wang and Schmid's trajectory settings (--descriptors, --fisher)
static ofdis_traj_params traj_settings() {
  ofdis_traj_params trp;
  memset(&trp, 0, sizeof(trp));
  trp.L = 15;
  trp.nt = 3;
  trp.N = 32;
  trp.ns = 2;
  trp.min_flow = 0.4f;
  trp.eps = 0.05f;
  trp.min_disp = 1.0f;
  trp.min_var = (float)std::sqrt(3.0);
  trp.max_var = 50.0f;
  trp.max_dis = 20.0f;
  return trp;
}

// Every flag's value as given, then what the checks read from them
struct Options {
  const char* batch = nullptr;  // --batch N: the last one given
  bool warm = false, bidir = false, kitti = false, color = false, lr_check = false, fill = false, mesh = false;
  const char* color_max_arg = nullptr;                // --color-max M
  const char* interp_arg = nullptr;                   // --interpolate T
  const char* gtlist = nullptr;                       // --gt gtlist
  const char* tracks = nullptr;                       // --tracks PATH
  const char* desc = nullptr;                         // --descriptors PATH
  const char* fisher[2] = {nullptr, nullptr};         // --fisher CODEBOOK PATH
  const char* speckle[2] = {nullptr, nullptr};        // --speckle N R
  const char* camera = nullptr;                       // --camera fx,fy,cx,cy,baseline,doffs
  const char* gm[2] = {nullptr, nullptr};             // --global-motion MODEL PATH
  const char* stab[3] = {nullptr, nullptr, nullptr};  // --stabilize RADIUS CROP DIR
  const char* sf_list = nullptr;                      // --scene-flow DISPLIST
  const char* sf_gtlist = nullptr;                    // --gt-scene-flow GTLIST
  const char* odo_dir = nullptr;                      // --odometry DIR
  const char* odo_gtlist = nullptr;                   // --gt-poses LIST
  const char* mono_dir = nullptr;                     // --mono-odometry DIR
  const char* intrinsics = nullptr;                   // --intrinsics fx,fy,cx,cy
  const char* fuse = nullptr;                         // --fuse voxel,trunc,x0,y0,z0,nx,ny,nz
  const char* conf_arg = nullptr;                     // --confidence R
  int nnum = 0;                                       // the operating point or the 20 parameters after the flags
  char** nums = nullptr;

  ofdis_relpose_params rpp{};  // --intrinsics: the parameters of --mono-odometry
  int maxb = 64;
  float color_max = 0.0f;   // 0: every pair's own maximum
  float interp_t = 0.0f;
  int gm_model = 0;         // OFDIS_MOTION_*
  bool disp_on = false;     // filtered disparities (stereo binaries)
  bool traj_stage = false;  // the descriptor stage runs in place of the tracker's calls
  bool two_way = false;     // the backward slots run
  ofdis_fuse_params fuse_p{};
  ofdis_traj_params trp = traj_settings();
  int tdim = 2 * trp.L + trp.ns * trp.ns * trp.nt * 33;  // floats per descriptor
  FisherBook fbook;  // --fisher: the codebook, whose blocks must be the descriptors' (shape, HOG, HOF, MBHx, MBHy)
  int fv_floats = 0;
  ofdis_stab_params stp{};
  vector<double> stab_wts;
  ofdis_disp_filter dfilt{};
  ofdis_stereo_camera dcam{};
  ofdis_conf_params cp{};
};

// The flags, read from argv[2] on until the first word that is none of them.  An argument-taking flag without its
// arguments, or given twice, is refused with what it takes; a switch may repeat.  --batch is the exception: a repeat
// keeps the last value, and a trailing --batch without one ends the flags (it is then read as the operating point).
static int parse_flags(int argc, char** argv, Options& o) {
  struct Flag {
    const char* name;
    int nargs;
    const char** dest;  // its nargs values
    bool* on;           // a switch
    const char* takes;  // nullptr: --batch
  };
  const Flag flags[] = {
      {"--batch", 1, &o.batch, nullptr, nullptr},
      {"--warm-start", 0, nullptr, &o.warm, nullptr},
      {"--bidirectional", 0, nullptr, &o.bidir, nullptr},
      {"--kitti", 0, nullptr, &o.kitti, nullptr},
      {"--color", 0, nullptr, &o.color, nullptr},
      {"--color-max", 1, &o.color_max_arg, nullptr, "one positive number"},
      {"--interpolate", 1, &o.interp_arg, nullptr, "one time between 0 and 1"},
      {"--tracks", 1, &o.tracks, nullptr, "one output path"},
      {"--descriptors", 1, &o.desc, nullptr, "one output path"},
      {"--fisher", 2, o.fisher, nullptr, "a codebook file and an output path"},
      {"--lr-check", 0, nullptr, &o.lr_check, nullptr},
      {"--fill", 0, nullptr, &o.fill, nullptr},
      {"--speckle", 2, o.speckle, nullptr, "a size N and a difference R"},
      {"--camera", 1, &o.camera, nullptr, "fx,fy,cx,cy,baseline,doffs"},
      {"--global-motion", 2, o.gm, nullptr, "a model (similarity, affine or homography) and an output path"},
      {"--stabilize", 3, o.stab, nullptr, "a radius, a crop and an output directory"},
      {"--scene-flow", 1, &o.sf_list, nullptr, "one disparity list file"},
      {"--gt-scene-flow", 1, &o.sf_gtlist, nullptr, "one ground-truth list file"},
      {"--odometry", 1, &o.odo_dir, nullptr, "one output directory"},
      {"--fuse", 1, &o.fuse, nullptr, "voxel,trunc,x0,y0,z0,nx,ny,nz"},
      {"--mesh", 0, nullptr, &o.mesh, nullptr},
      {"--gt-poses", 1, &o.odo_gtlist, nullptr, "one list of KITTI poses files"},
      {"--mono-odometry", 1, &o.mono_dir, nullptr, "one output directory"},
      {"--intrinsics", 1, &o.intrinsics, nullptr, "fx,fy,cx,cy"},
      {"--gt", 1, &o.gtlist, nullptr, "one ground-truth list file"},
      {"--confidence", 1, &o.conf_arg, nullptr, "one window radius"},
  };
  int i = 2;
  while (i < argc) {
    const Flag* f = nullptr;
    for (const Flag& g : flags)
      if (!strcmp(argv[i], g.name)) f = &g;
    if (!f) break;
    const bool missing = i + f->nargs >= argc;
    if (!f->takes && missing) break;
    if (f->takes && (missing || f->dest[0])) return refuse(2, "%s takes %s", f->name, f->takes);
    if (f->on) *f->on = true;
    for (int a = 0; a < f->nargs; ++a) f->dest[a] = argv[i + 1 + a];
    i += 1 + f->nargs;
  }
  o.nnum = argc - i;
  o.nums = argv + i;
  return 0;
}

// The value readers of the flags that take numbers, a model or a codebook: each refuses a bad value
static int read_fuse(Options& o) {
  double v[8];
  const char* q = o.fuse;
  bool ok = true;
  for (int i = 0; i < 8 && ok; ++i) {
    char* end = nullptr;
    v[i] = strtod(q, &end);
    ok = end != q && (i < 7 ? *end == ',' : *end == 0) && std::isfinite(v[i]);
    q = end + (i < 7 ? 1 : 0);
  }
  for (int i = 5; i < 8 && ok; ++i) ok = v[i] >= 1.0 && v[i] <= (double)(1 << 30) && v[i] == std::floor(v[i]);
  ok = ok && (float)v[0] > 0.0f && (float)v[1] > 0.0f && v[0] <= FLT_MAX && v[1] <= FLT_MAX &&
       std::fabs(v[2]) <= FLT_MAX && std::fabs(v[3]) <= FLT_MAX && std::fabs(v[4]) <= FLT_MAX &&
       v[5] * v[6] * v[7] <= (double)(1 << 30);
  if (!ok)
    return refuse(2, "--fuse takes eight numbers voxel,trunc,x0,y0,z0,nx,ny,nz with voxel and trunc > 0, integer sizes "
                     ">= 1 and at most 2^30 voxels, got %s", o.fuse);
  o.fuse_p.voxel = (float)v[0];
  o.fuse_p.trunc = (float)v[1];
  for (int e = 0; e < 3; ++e) o.fuse_p.origin[e] = (float)v[2 + e];
  o.fuse_p.nx = (int)v[5];
  o.fuse_p.ny = (int)v[6];
  o.fuse_p.nz = (int)v[7];
  o.fuse_p.max_weight = 64.0f;
  o.fuse_p.color = 1;
  return 0;
}

static int read_global_motion(Options& o) {
  o.gm_model = !strcmp(o.gm[0], "similarity")   ? OFDIS_MOTION_SIMILARITY
               : !strcmp(o.gm[0], "affine")     ? OFDIS_MOTION_AFFINE
               : !strcmp(o.gm[0], "homography") ? OFDIS_MOTION_HOMOGRAPHY : 0;
  if (!o.gm_model) return refuse(2, "--global-motion takes the model similarity, affine or homography, got %s", o.gm[0]);
  return 0;
}

static int read_codebook(Options& o) {
  string err;
  if (!read_fisher_book(o.fisher[0], o.fbook, err)) return refuse(2, "%s: %s", o.fisher[0], err.c_str());
  const ofdis_traj_params& t = o.trp;
  const int c = t.nt * t.ns * t.ns, din[5] = {2 * t.L, 8 * c, 9 * c, 8 * c, 8 * c};
  const ofdis_fisher_codebook& cb = o.fbook.cb;
  bool match = cb.desc_dim == o.tdim && cb.nblocks == 5;
  for (int b = 0, off = 0; match && b < 5; off += din[b++])
    match = cb.blocks[b].offset == off && cb.blocks[b].dim_in == din[b];
  if (!match)
    return refuse(2, "%s: the codebook's blocks are not the descriptors' (desc_dim %d, blocks 0+%d, %d+%d, %d+%d, %d+%d, "
                     "%d+%d)", o.fisher[0], o.tdim, din[0], din[0], din[1], din[0] + din[1], din[2],
                  din[0] + din[1] + din[2], din[3], o.tdim - din[4], din[4]);
  for (int b = 0; b < cb.nblocks; ++b) o.fv_floats += 2 * cb.K * cb.blocks[b].dim;
  return 0;
}

static int read_stabilize(Options& o) {
  char *e0 = nullptr, *e1 = nullptr;
  const long r = strtol(o.stab[0], &e0, 10);
  const float crop = strtof(o.stab[1], &e1);
  if (e0 == o.stab[0] || *e0 || r < 1 || r > 64 || e1 == o.stab[1] || *e1 || !(crop >= 0.0f && crop < 0.5f))
    return refuse(2, "--stabilize takes a radius 1..64 and a crop 0 <= CROP < 0.5, got %s %s", o.stab[0], o.stab[1]);
  o.stp.radius = (int)r;
  o.stp.crop = crop;
  o.stp.limit = crop > 0.0f ? 1 : 0;
  for (int d = 0; d <= o.stp.radius; ++d) o.stab_wts.push_back(exp(-(double)(d * d) / (2.0 * o.stp.radius)));
  return 0;
}

static int read_speckle(Options& o) {
  char *e0 = nullptr, *e1 = nullptr;
  const long sz = strtol(o.speckle[0], &e0, 10);
  const float diff = strtof(o.speckle[1], &e1);
  if (e0 == o.speckle[0] || *e0 || sz < 1 || sz > INT_MAX || e1 == o.speckle[1] || *e1 ||
      !(diff >= 0.0f && diff <= FLT_MAX))
    return refuse(2, "--speckle takes a size N >= 1 and a finite difference R >= 0, got %s %s", o.speckle[0],
                  o.speckle[1]);
  o.dfilt.speckle_size = (int)sz;
  o.dfilt.speckle_diff = diff;
  return 0;
}

static int read_camera(Options& o) {
  float v[6];
  const char* q = o.camera;
  bool ok = true;
  for (int i = 0; i < 6 && ok; ++i) {
    char* end = nullptr;
    v[i] = strtof(q, &end);
    ok = end != q && (i < 5 ? *end == ',' : *end == 0) && v[i] >= -FLT_MAX && v[i] <= FLT_MAX;
    q = end + (i < 5 ? 1 : 0);
  }
  if (!ok || !(v[0] > 0.0f) || !(v[1] > 0.0f) || !(v[4] > 0.0f))
    return refuse(2, "--camera takes six finite numbers fx,fy,cx,cy,baseline,doffs with fx, fy and baseline > 0, got %s",
                  o.camera);
  o.dcam = ofdis_stereo_camera{v[0], v[1], v[2], v[3], v[4], v[5]};
  return 0;
}

static int read_intrinsics(Options& o) {
  float v[4];
  const char* q = o.intrinsics;
  bool ok = true;
  for (int i = 0; i < 4 && ok; ++i) {
    char* end = nullptr;
    v[i] = strtof(q, &end);
    ok = end != q && (i < 3 ? *end == ',' : *end == 0) && v[i] >= -FLT_MAX && v[i] <= FLT_MAX;
    q = end + (i < 3 ? 1 : 0);
  }
  if (!ok || !(v[0] > 0.0f) || !(v[1] > 0.0f))
    return refuse(2, "--intrinsics takes four finite numbers fx,fy,cx,cy with fx and fy > 0, got %s", o.intrinsics);
  memset(&o.rpp, 0, sizeof(o.rpp));
  o.rpp.fx = v[0], o.rpp.fy = v[1], o.rpp.cx = v[2], o.rpp.cy = v[3];
  o.rpp.step = 8;
  o.rpp.alpha = 0.01f;
  o.rpp.beta = 0.5f;
  o.rpp.hypotheses = 1024;
  o.rpp.threshold = 1.0f;
  o.rpp.refine = 5;
  o.rpp.min_parallax = 0.5f;
  o.rpp.seed = 0;
  return 0;
}

static int read_interpolate(Options& o) {
  char* end = nullptr;
  o.interp_t = strtof(o.interp_arg, &end);
  if (end == o.interp_arg || *end || !(o.interp_t > 0.0f && o.interp_t < 1.0f))
    return refuse(2, "--interpolate takes a time T with 0 < T < 1, got %s", o.interp_arg);
  return 0;
}

static int read_confidence(Options& o) {
  char* end = nullptr;
  const long r = strtol(o.conf_arg, &end, 10);
  if (end == o.conf_arg || *end || r < 1 || r > 7) return refuse(2, "--confidence takes a radius 1..7, got %s", o.conf_arg);
  const int side = 2 * (int)r + 1;
  o.cp = ofdis_conf_params{(int)r, 1.0f, 100.0f, side * side / 2};
  return 0;
}

static int read_color_max(Options& o) {
  char* end = nullptr;
  o.color_max = strtof(o.color_max_arg, &end);
  if (end == o.color_max_arg || *end || !(o.color_max > 0.0f && o.color_max <= FLT_MAX))
    return refuse(2, "--color-max takes a positive finite number, got %s", o.color_max_arg);
  return 0;
}

// The option refusals, before any file is read: the rules in order, the first that fails refuses the run (exit 2).
// Each rule is one given flag: the binaries of the other kind refuse it, saying what it does; --warm-start, which
// runs one pair per launch, refuses it; it needs another flag; then its value is read.
static int check_options(Options& o) {
  enum { kAny, kFlow, kStereo };
  struct Rule {
    bool given;
    const char* flag;  // as the refusals name it
    int only;          // kFlow, kStereo: what it does, which the other binaries are told
    const char* does;
    bool no_warm;
    bool has_needed;  // false: refused with `needs`
    const char* needs;
    int (*value)(Options&);
  };
  o.disp_on = o.lr_check || o.fill || o.speckle[0] || (o.camera && !o.sf_list);  // --camera with --scene-flow is its own
  o.dfilt.lr_check = o.lr_check ? 1 : 0;
  o.dfilt.alpha = 0.0f;
  o.dfilt.beta = 1.0f;
  o.dfilt.speckle_diff = 1.0f;
  o.dfilt.fill = o.fill ? 1 : 0;
  const Rule rules[] = {
      {o.batch != nullptr, "--batch", kAny, nullptr, true, true, nullptr, nullptr},
      {o.bidir, "--bidirectional", kAny, nullptr, true, true, nullptr, nullptr},
      {o.interp_arg != nullptr, "--interpolate", kAny, nullptr, true, true, nullptr, nullptr},
      {o.tracks != nullptr, "--tracks", kAny, nullptr, true, true, nullptr, nullptr},
      {o.sf_list != nullptr, "--scene-flow", kFlow, "--scene-flow joins flows with disparities", true, true, nullptr,
       nullptr},
      {o.sf_gtlist != nullptr, "--gt-scene-flow", kAny, nullptr, false, o.sf_list != nullptr,
       "--gt-scene-flow evaluates the scene flow of --scene-flow; give --scene-flow too", nullptr},
      {o.odo_dir != nullptr, "--odometry", kFlow, "--odometry fits the rig's motion from flows", true,
       o.sf_list && o.camera, "--odometry needs the disparities of --scene-flow and the stereo camera of --camera",
       nullptr},
      {o.mono_dir != nullptr, "--mono-odometry", kFlow, "--mono-odometry fits the camera's motion from flows", true,
       o.intrinsics != nullptr, "--mono-odometry needs the camera intrinsics of --intrinsics", nullptr},
      {o.intrinsics != nullptr, "--intrinsics", kFlow, "--intrinsics calibrates the camera of --mono-odometry", true,
       o.mono_dir != nullptr, "--intrinsics calibrates the camera of --mono-odometry; give --mono-odometry too",
       read_intrinsics},
      {o.odo_gtlist != nullptr, "--gt-poses", kAny, nullptr, false, o.odo_dir != nullptr || o.mono_dir != nullptr,
       "--gt-poses evaluates the poses of --odometry; give --odometry too", nullptr},
      {o.fuse != nullptr, "--fuse", kFlow, "--fuse places disparities with the poses of --odometry", true,
       o.odo_dir != nullptr, "--fuse places disparities with the poses of --odometry; give --odometry too", read_fuse},
      {o.mesh, "--mesh", kAny, nullptr, false, o.fuse != nullptr, "--mesh meshes the volume of --fuse; give --fuse too",
       nullptr},
      {o.disp_on, "--lr-check, --speckle, --fill or --camera", kStereo,
       "--lr-check, --speckle, --fill and --camera filter stereo disparities", true, true, nullptr, nullptr},
      {o.gm[0] != nullptr, "--global-motion", kFlow, "--global-motion fits the camera motion of flows", true, true,
       nullptr, read_global_motion},
      {o.desc != nullptr, "--descriptors", kFlow, "--descriptors describes the tracks of flows", true,
       o.tracks != nullptr, "--descriptors describes the clips of --tracks; give --tracks too", nullptr},
      {o.fisher[0] != nullptr, "--fisher", kFlow, "--fisher encodes the descriptors of flows", true,
       o.tracks != nullptr, "--fisher encodes the clips of --tracks; give --tracks too", read_codebook},
      {o.stab[0] != nullptr, "--stabilize", kFlow, "--stabilize smooths the camera motion of flows", true,
       o.gm[0] != nullptr, "--stabilize smooths the models of --global-motion; give --global-motion too",
       read_stabilize},
      {o.speckle[0] != nullptr, "--speckle", kAny, nullptr, false, true, nullptr, read_speckle},
      {o.camera != nullptr, "--camera", kAny, nullptr, false, true, nullptr, read_camera},
      {o.interp_arg != nullptr, "--interpolate", kAny, nullptr, false, true, nullptr, read_interpolate},
      {o.color_max_arg != nullptr, "--color-max", kAny, nullptr, false, o.color, "--color-max needs --color",
       read_color_max},
      {o.conf_arg != nullptr, "--confidence", kAny, nullptr, true, true, nullptr, read_confidence},
  };
  for (const Rule& r : rules) {
    if (!r.given) continue;
    if (r.only == kFlow && SELECTMODE != 1) return refuse(2, "%s; the stereo binaries take no %s", r.does, r.flag);
    if (r.only == kStereo && SELECTMODE == 1) return refuse(2, "%s; the flow binaries take none of them", r.does);
    if (r.no_warm && o.warm) return refuse(2, "--warm-start runs one pair per launch; it takes no %s", r.flag);
    if (!r.has_needed) return refuse(2, "%s", r.needs);
    if (r.value)
      if (int rc = r.value(o)) return rc;
  }
  o.traj_stage = o.desc || o.fisher[0];
  // --interpolate and --tracks need the backward flows: the backward slots run whenever one of them is given
  o.two_way = o.bidir || o.interp_arg || o.tracks || o.lr_check;
  o.maxb = o.warm ? 1 : o.batch ? atoi(o.batch) : 64;
  if (o.maxb < 1 || (o.nnum > 1 && o.nnum != 20))
    return refuse(2, "expected 0, 1 or exactly 20 numbers, got %d", o.nnum);
  return 0;
}

struct Job {
  string a, b, out;
};

static int refuse_pair(const Job& jb) {
  return refuse(1, "cannot read the pair %s %s (binary PGM/PPM or 8-bit PNG of equal size)", jb.a.c_str(),
                jb.b.c_str());
}

// The clip index: pair k continues pair k - 1 when its image1 path is pair k - 1's image2 path (string equality).
// clip[k] and frame[k] count from 0; a pair of frame 0 begins its clip.
struct ClipIndex {
  vector<int> clip, frame;
  int count = 0;
};

static ClipIndex index_clips(const vector<Job>& jobs) {
  ClipIndex ci;
  for (size_t k = 0; k < jobs.size(); ++k) {
    const bool cont = k > 0 && jobs[k].a == jobs[k - 1].b;
    ci.clip.push_back(cont ? ci.clip[k - 1] : ci.count++);
    ci.frame.push_back(cont ? ci.frame[k - 1] + 1 : 0);
  }
  return ci;
}

// A batch's pairs [k0, k1) of one clip, whether they begin it and whether they end it
struct ClipRun {
  int k0, k1;
  bool starts, ends;
};

static vector<ClipRun> clip_runs(const ClipIndex& ci, size_t j0, int n) {
  vector<ClipRun> runs;
  for (int k0 = 0, k1; k0 < n; k0 = k1) {
    for (k1 = k0 + 1; k1 < n && ci.frame[j0 + k1] > 0;) ++k1;
    runs.push_back({k0, k1, ci.frame[j0 + k0] == 0, j0 + k1 == ci.frame.size() || ci.frame[j0 + k1] == 0});
  }
  return runs;
}

// The per-pair input lists, every file checked against its pair's image size before any device work
struct Inputs {
  vector<string> gts;               // --gt: one per pair
  vector<string> sf_files, sf_gts;  // --scene-flow: two per pair; --gt-scene-flow: three
  vector<vector<double>> odo_gt;    // --gt-poses: per clip, 12 numbers per line
};

static int read_inputs(const Options& o, const vector<Job>& jobs, const ClipIndex& clips, Inputs& in) {
  const int nop = SELECTMODE == 1 ? 2 : 1;
  vector<float> tmp;
  string err;
  int iw = 0, ih = 0;
  if (o.gtlist) {
    if (!read_words(o.gtlist, in.gts)) return refuse(1, "cannot read %s", o.gtlist);
    if (in.gts.size() != jobs.size())
      return refuse(2, "--gt: %s lists %zu ground-truth files for %zu pairs", o.gtlist, in.gts.size(), jobs.size());
    for (size_t k = 0; k < jobs.size(); ++k) {
      if (!image_size(jobs[k].a.c_str(), iw, ih)) return refuse_pair(jobs[k]);
      if (!read_gt_file(in.gts[k].c_str(), iw, ih, nop, tmp, err))
        return refuse(1, "%s: %s", in.gts[k].c_str(), err.c_str());
    }
  }
  for (int li = 0; li < 2; ++li) {  // --scene-flow, --gt-scene-flow
    const char* list = li ? o.sf_gtlist : o.sf_list;
    vector<string>& files = li ? in.sf_gts : in.sf_files;
    const size_t per = li ? 3 : 2;
    if (!list) continue;
    if (!read_words(list, files)) return refuse(1, "cannot read %s", list);
    if (files.size() != per * jobs.size())
      return refuse(2, "%s: %s lists %zu files for %zu pairs (%zu per pair)", li ? "--gt-scene-flow" : "--scene-flow",
                    list, files.size(), jobs.size(), per);
    for (size_t k = 0; k < files.size(); ++k) {
      if (!image_size(jobs[k / per].a.c_str(), iw, ih)) return refuse_pair(jobs[k / per]);
      if (!read_gt_file(files[k].c_str(), iw, ih, li && k % 3 == 2 ? 2 : 1, tmp, err))
        return refuse(2, "%s: %s", files[k].c_str(), err.c_str());
    }
  }
  if (o.odo_gtlist) {  // a poses file per clip, with a line for each of its frames
    vector<string> files;
    if (!read_words(o.odo_gtlist, files)) return refuse(2, "cannot read %s", o.odo_gtlist);
    if ((int)files.size() != clips.count)
      return refuse(2, "--gt-poses: %s lists %zu poses files for %d clips", o.odo_gtlist, files.size(), clips.count);
    vector<int> need(clips.count, 0);
    for (size_t k = 0; k < jobs.size(); ++k) need[clips.clip[k]] = clips.frame[k] + 2;
    for (int c = 0; c < clips.count; ++c) {
      FILE* pf = fopen(files[c].c_str(), "r");
      if (!pf) return refuse(2, "cannot read %s", files[c].c_str());
      vector<double> v;
      double x;
      while (fscanf(pf, "%lf", &x) == 1) v.push_back(x);
      const bool eof = feof(pf);
      fclose(pf);
      if (!eof || v.size() % 12 || (int)(v.size() / 12) < need[c])
        return refuse(2, "%s: a KITTI poses file of at least %d lines of 12 numbers, got %zu numbers",
                      files[c].c_str(), need[c], v.size());
      in.odo_gt.push_back(v);
    }
  }
  return 0;
}

// The list outputs, one file each for the whole run
struct ListOutputs {
  struct File {
    FILE* f = nullptr;
    string path;
  };
  File odo, desc, fisher, tracks, stab, gm, mono;

  bool open(File& x, const string& path) {
    x.path = path;
    x.f = fopen(path.c_str(), "w");
    return x.f != nullptr;
  }
  // The end of a run: stab.txt, tracks, descriptors, fisher, global motion and odometry.txt are closed in this order,
  // and the first that cannot be written is refused
  int close() {
    for (File* x : {&stab, &tracks, &desc, &fisher, &gm, &odo, &mono}) {
      if (!x->f) continue;
      const bool ok = fclose(x->f) == 0;
      x->f = nullptr;
      if (!ok) return refuse(1, "cannot write %s", x->path.c_str());
    }
    return 0;
  }
  ~ListOutputs() {  // a refused run
    for (File* x : {&stab, &tracks, &desc, &fisher, &gm, &odo, &mono})
      if (x->f) fclose(x->f);
  }
};

// Opened before any device work in this order, which decides the files a refused run leaves behind: odometry.txt,
// descriptors, fisher, tracks, stab.txt, global motion.  The descriptor stage's frame sizes are checked after
// odometry.txt is opened.
static int open_outputs(const Options& o, const vector<Job>& jobs, ListOutputs& out) {
  if (o.odo_dir && !out.open(out.odo, string(o.odo_dir) + "/odometry.txt"))
    return refuse(2, "--odometry: cannot write %s", out.odo.path.c_str());
  if (o.mono_dir && !out.open(out.mono, string(o.mono_dir) + "/monodometry.txt"))
    return refuse(2, "--mono-odometry: cannot write %s", out.mono.path.c_str());
  for (size_t k = 0; k < jobs.size() && o.traj_stage; ++k) {  // an N x N patch in every frame
    int iw = 0, ih = 0;
    if (!image_size(jobs[k].a.c_str(), iw, ih)) return refuse_pair(jobs[k]);
    if (iw < o.trp.N || ih < o.trp.N)
      return refuse(2, "--%s needs frames of at least %d x %d, %s is %d x %d", o.desc ? "descriptors" : "fisher",
                    o.trp.N, o.trp.N, jobs[k].a.c_str(), iw, ih);
  }
  if (o.desc) {
    if (!out.open(out.desc, o.desc)) return refuse(1, "cannot write %s", o.desc);
    fprintf(out.desc.f, "# clip id start mean_x mean_y sd_x sd_y length d0 .. d%d\n", o.tdim - 1);
  }
  if (o.fisher[0]) {
    if (!out.open(out.fisher, o.fisher[1])) return refuse(1, "cannot write %s", o.fisher[1]);
    fprintf(out.fisher.f, "# clip n_desc n_0 .. n_%d fv0 .. fv%d\n", o.fbook.cb.nblocks - 1, o.fv_floats - 1);
  }
  if (o.tracks) {
    if (!out.open(out.tracks, o.tracks)) return refuse(1, "cannot write %s", o.tracks);
    fprintf(out.tracks.f, "# clip frame id x y\n");
  }
  if (o.stab[0] && !out.open(out.stab, string(o.stab[2]) + "/stab.txt"))
    return refuse(1, "cannot write %s", out.stab.path.c_str());
  if (o.gm_model && !out.open(out.gm, o.gm[1])) return refuse(1, "cannot write %s", o.gm[1]);
  return 0;
}

struct CtxDeleter {
  void operator()(ofdis_ctx* c) const { ofdis_destroy(c); }
};

// One batch: pairs j0 .. j0 + n - 1 of one size, their frames, and what the device stages return for them
struct Batch {
  size_t j0 = 0;
  int n = 0, w = 0, h = 0, slots = 0;
  bool seq = false;  // a clip: frame k is image1 of pair k, frame k + 1 its image2
  size_t hwc = 0;    // bytes per frame
  size_t fs = 0;     // image1 of pair k at k * fs, its image2 one frame (hwc) later
  vector<uint8_t> frames;
  vector<float> flows;
  vector<uint16_t> kflows;  // --kitti: the encoded slots
  vector<uint8_t> masks;
  vector<uint8_t> colors;  // --color: the color images of the slots
  vector<uint8_t> interp;  // --interpolate: the frames at time T
  vector<float> ddisp, ddepth, dxyz;  // --lr-check / --speckle / --fill / --camera: the filtered outputs
  vector<uint8_t> dstatus;
  size_t dcount[6];  // statuses 0..4, filled
  vector<double> gm_models;  // --global-motion: the models, stats and per-pixel outputs
  vector<ofdis_motion_stats> gm_stats;
  vector<uint8_t> gm_mask, gm_reg;
  vector<float> gm_res;
  vector<float> sf_d0, sf_d1, sf_w, sf_m;  // --scene-flow: the disparities of image1 and image2, outputs
  vector<double> odo_pose;                 // --odometry: the relative poses
  vector<float> conf;                      // --confidence: the forward slots' confidence maps
};

// The run's state across batches: the context and what clips and the end-of-run summary carry over
struct State {
  State(const Options& o_, const vector<Job>& jobs_, const ClipIndex& clips_, const Inputs& in_, ListOutputs& out_)
      : o(o_), jobs(jobs_), clips(clips_), in(in_), out(out_), nclasses(o_.bidir ? 3 : 1), eval_total(nclasses + 1),
        sf_total(nclasses + 1), fvec(o_.fv_floats) {
    memset(eval_total.data(), 0, sizeof(ofdis_error_stats) * eval_total.size());
    memset(sf_total.data(), 0, sizeof(ofdis_sf_stats) * sf_total.size());
    if (o.odo_dir) odo_rel.resize(clips.count);
    if (o.mono_dir) mono_rel.resize(clips.count);
  }
  const Options& o;
  const vector<Job>& jobs;
  const ClipIndex& clips;
  const Inputs& in;
  ListOutputs& out;
  const int nochannels = SELECTCHANNEL == 3 ? 3 : 1, nop = SELECTMODE == 1 ? 2 : 1;
  const int nclasses;  // with --bidirectional the forward consistency mask's classes
  std::unique_ptr<ofdis_ctx, CtxDeleter> ctx;
  int ctx_w = -1, ctx_h = -1, verbosity = 0;
  Image8 last;  // image2 of the previous batch's last pair
  size_t done = 0, seq_pairs = 0, seq_decoded = 0, warm_pairs = 0;
  vector<ofdis_error_stats> eval_total;  // --gt: [0] all pixels, [1 + c] class c
  vector<ofdis_sf_stats> sf_total;       // --gt-scene-flow, as eval_total
  // --tracks: the clip being tracked (-1 none) and its next frame; the totals of the finished clips (with
  // --descriptors and --fisher theirs too)
  int tclip = -1, tframe = 0;
  size_t tframes = 0;
  ofdis_track_stats ttotal{};
  ofdis_traj_stats dtotal{};
  vector<float> fvec;
  int fclips = 0;
  long long fpushed = 0, fskipped[OFDIS_FISHER_MAX_BLOCKS] = {0};
  int sclip = -1;  // --stabilize: the clip being stabilised (-1 none)
  vector<vector<double>> odo_rel;  // --odometry: per clip, 12 numbers per pair
  vector<vector<double>> mono_rel;  // --mono-odometry: per clip, 12 numbers per pair (|t| = 1)
  double mono_rerr = 0.0, mono_terr = 0.0;
  size_t mono_eval = 0;
  vector<ofdis_motion_stats> mono_stats;
  vector<double> mono_pose;
  vector<uint8_t> mono_mask;
  vector<float> mono_depth;
  double odo_terr = 0.0, odo_rerr = 0.0;
  size_t odo_eval = 0;
  double fuse_T[12];    // --fuse: the chained pose of the clip's next image1
  int fuse_frames = 0;  // frames pushed into the clip's volume
  // scratch of the stages, kept across batches
  vector<uint8_t> png;
  vector<float> gt_batch, gt_one;
  vector<ofdis_error_stats> eval_pairs;
  vector<float> sf_g0, sf_g1, sf_gf;
  vector<ofdis_sf_stats> sf_pairs;
  vector<ofdis_motion_stats> odo_stats;
  vector<uint8_t> odo_mask;
  vector<float> odo_om;
  vector<ofdis_track_point> tpoints;
  vector<int> tcounts, tndesc;
  vector<ofdis_traj_record> trec;
  vector<float> tdesc;
  vector<uint8_t> sbuf;
  vector<ofdis_stab_frame> sinfo;
  vector<double> fuse_poses;
  vector<ofdis_fuse_point> fuse_pts;
  vector<unsigned int> fuse_faces;
};

// Up to maxb pairs of one size from pair j0 on; a frame that continues the previous pair is not decoded again.  A
// batch of two or more pairs that all continue each other is a clip and goes up frame by frame; any other batch goes
// as its pairs, followed with two_way by their swapped copies.
static int load_batch(State& s, Batch& b, size_t j0) {
  const vector<Job>& jobs = s.jobs;
  vector<Image8> imgs;  // decoded frames of this batch
  vector<int> ia, ib;   // per pair: indices of image1, image2 in imgs
  int w = 0, h = 0, n = 0, decoded = 0;
  while (j0 + n < jobs.size() && n < s.o.maxb) {
    const Job& jb = jobs[j0 + n];
    const bool in_batch = n > 0 && jb.a == jobs[j0 + n - 1].b;          // image1 = this batch's last frame
    const bool from_last = n == 0 && j0 > 0 && jb.a == jobs[j0 - 1].b;  // image1 = the previous batch's last frame
    Image8 a8, b8;
    if (from_last) a8 = s.last;
    const bool ok = in_batch || from_last || load_image(jb.a.c_str(), s.nochannels, a8);
    const Image8& ra = in_batch ? imgs[ib.back()] : a8;
    if (!ok || !load_image(jb.b.c_str(), s.nochannels, b8) || ra.w != b8.w || ra.h != b8.h) return refuse_pair(jb);
    if (n == 0) {
      w = b8.w;
      h = b8.h;
    } else if (b8.w != w || b8.h != h) {
      break;  // next group
    }
    if (in_batch) {
      ia.push_back(ib.back());
    } else {
      decoded += from_last ? 0 : 1;
      ia.push_back((int)imgs.size());
      imgs.push_back(std::move(a8));
    }
    ib.push_back((int)imgs.size());
    imgs.push_back(std::move(b8));
    ++decoded;
    ++n;
  }
  b.j0 = j0;
  b.n = n;
  b.w = w;
  b.h = h;
  b.hwc = (size_t)w * h * s.nochannels;
  b.seq = n >= 2;
  for (int k = 1; k < n && b.seq; ++k) b.seq = ia[k] == ib[k - 1];
  b.fs = b.seq ? b.hwc : 2 * b.hwc;
  b.slots = s.o.two_way ? 2 * n : n;  // two-way: forward slots [0, n), backward slots [n, 2n)
  auto put = [&b, &imgs](int i) { b.frames.insert(b.frames.end(), imgs[i].px.begin(), imgs[i].px.end()); };
  b.frames.clear();
  if (b.seq) {
    put(ia[0]);
    for (int k = 0; k < n; ++k) put(ib[k]);
    s.seq_pairs += n;
    s.seq_decoded += decoded;
  } else {
    for (int k = 0; k < n; ++k) {
      put(ia[k]);
      put(ib[k]);
    }
    for (int k = 0; k < n && s.o.two_way; ++k) {  // the swapped copies
      put(ib[k]);
      put(ia[k]);
    }
  }
  s.last = std::move(imgs[ib.back()]);
  return 0;
}

// A context per frame size.  The clip-scoped stages (the tracker or the descriptor stage, the Fisher encoder, the
// stabiliser, the fusion volume) keep a clip's state in the context, so every clip must end before its context is
// destroyed.  It does: a size change always begins a clip (a pair that continues the previous one shares its frame),
// and each of these stages ends a clip with the run of pairs that ends it, in the batch that holds that run.
static int ensure_context(State& s, const Batch& b, const CliParams& P) {
  if (b.w == s.ctx_w && b.h == s.ctx_h) return 0;
  s.ctx.reset();
  ofdis_params p;
  memset(&p, 0, sizeof(p));
  p.sc_f = P.lv_f; p.sc_l = P.lv_l; p.max_iter = P.maxiter; p.min_iter = P.miniter;
  p.dp_thresh = P.mindprate; p.dr_thresh = P.mindrrate; p.res_thresh = P.minimgerr;
  p.p_samp_s = P.patchsz; p.patove = P.poverl; p.usefbcon = P.usefbcon ? 1 : 0; p.costfct = P.costfct;
  p.noc = s.nochannels; p.patnorm = P.patnorm; p.usetvref = P.usetvref ? 1 : 0;
  p.tv_alpha = P.tv_alpha; p.tv_gamma = P.tv_gamma; p.tv_delta = P.tv_delta;
  p.tv_innerit = P.tv_innerit; p.tv_solverit = P.tv_solverit; p.tv_sor = P.tv_sor; p.verbosity = P.verbosity;
  const int scf = 1 << (s.o.warm ? P.lv_f + 1 : P.lv_f);
  ofdis_ctx* ctx = nullptr;
  const int rc = ofdis_create(&ctx, 0, nullptr, &p, s.nop, (b.w + scf - 1) / scf * scf, (b.h + scf - 1) / scf * scf,
                              P.patchsz, s.o.two_way ? 2 * s.o.maxb : s.o.maxb);
  if (rc != OFDIS_OK) return refuse(1, "ofdis_create failed with status %d for %dx%d frames", rc, b.w, b.h);
  s.ctx.reset(ctx);
  ofdis_set_graph_mode(ctx, 1);
  s.ctx_w = b.w;
  s.ctx_h = b.h;
  return 0;
}

// The flows of the batch's slots, with --color their colors and with --bidirectional the consistency masks
static int run_flows(State& s, Batch& b) {
  const Options& o = s.o;
  ofdis_ctx* ctx = s.ctx.get();
  const int n = b.n, w = b.w, h = b.h;
  if (o.kitti) b.kflows.resize((size_t)b.slots * w * h * (s.nop == 2 ? 3 : 1));
  else b.flows.resize((size_t)b.slots * w * h * s.nop);
  int rc;
  if (o.two_way && b.seq) {
    rc = ofdis_upload_sequence_bidir_u8(ctx, 0, n, b.frames.data(), w, h, OFDIS_MEM_HOST);
  } else if (o.two_way) {
    rc = ofdis_upload_frames_u8(ctx, 0, 2 * n, b.frames.data(), w, h, OFDIS_MEM_HOST);
    if (rc == OFDIS_OK) rc = ofdis_set_swapped_slots(ctx, 0, n, 0);
    if (rc == OFDIS_OK) rc = ofdis_set_swapped_slots(ctx, n, 2 * n, 1);
  } else {
    rc = b.seq ? ofdis_upload_sequence_u8(ctx, 0, n, b.frames.data(), w, h, OFDIS_MEM_HOST)
               : ofdis_upload_frames_u8(ctx, 0, n, b.frames.data(), w, h, OFDIS_MEM_HOST);
  }
  // warm start: the context still holds the previous pair's flow (same size, so it was not recreated)
  const bool from_prev = o.warm && s.clips.frame[b.j0] > 0;
  if (rc == OFDIS_OK && from_prev) rc = ofdis_set_initflow_from_result(ctx, 0, 1, 0, w, h);
  s.warm_pairs += from_prev ? 1 : 0;
  if (rc == OFDIS_OK) rc = ofdis_run(ctx, b.slots, from_prev ? 1 : 0);
  if (rc == OFDIS_OK)
    rc = o.kitti ? ofdis_get_flow_fullres_encoded(ctx, 0, b.slots, OFDIS_ENC_KITTI, b.kflows.data(), w, h, OFDIS_MEM_HOST)
                 : ofdis_get_flow_fullres(ctx, 0, b.slots, b.flows.data(), w, h, OFDIS_MEM_HOST);
  if (rc == OFDIS_OK && o.color) {
    b.colors.resize((size_t)b.slots * w * h * 3);
    rc = ofdis_flow_color_fullres(ctx, 0, b.slots, b.colors.data(), nullptr, o.color_max, w, h, OFDIS_MEM_HOST);
  }
  if (rc == OFDIS_OK && o.bidir) {
    b.masks.resize((size_t)n * w * h);
    rc = ofdis_consistency_fullres(ctx, 0, n, n, b.masks.data(), nullptr, s.nop == 2 ? 0.01f : 0.0f,
                                   s.nop == 2 ? 0.5f : 1.0f, w, h, OFDIS_MEM_HOST);
  }
  return rc;
}

// --interpolate: image1 / image2 of pair k are frames k and k + 1 of a clip, or the k-th pair of the pairs layout
static int run_interpolate(State& s, Batch& b) {
  b.interp.resize((size_t)b.n * b.hwc);
  return ofdis_interpolate_fullres(s.ctx.get(), 0, b.n, b.n, b.frames.data(), b.frames.data() + b.hwc, b.fs,
                                   s.o.interp_t, s.nop == 2 ? 0.01f : 0.0f, s.nop == 2 ? 0.5f : 1.0f, b.interp.data(),
                                   nullptr, b.w, b.h, OFDIS_MEM_HOST);
}

// --confidence: the forward slots' maps, with the forward-backward term when the backward slots run
static int run_confidence(State& s, Batch& b) {
  b.conf.resize((size_t)b.n * b.w * b.h);
  return ofdis_confidence_fullres(s.ctx.get(), 0, b.n, s.o.two_way ? b.n : -1, &s.o.cp, b.frames.data(),
                                  b.frames.data() + b.hwc, b.fs, b.conf.data(), nullptr, b.w, b.h, OFDIS_MEM_HOST);
}

static int run_global_motion(State& s, Batch& b) {
  const size_t np = (size_t)b.n * b.w * b.h;
  b.gm_models.resize((size_t)9 * b.n);
  b.gm_stats.resize(b.n);
  b.gm_mask.resize(np);
  b.gm_res.resize(2 * np);
  b.gm_reg.resize((size_t)b.n * b.hwc);
  ofdis_motion_params mp;
  memset(&mp, 0, sizeof(mp));
  mp.model = s.o.gm_model;
  mp.step = 8;
  mp.fb_check = s.o.bidir ? 1 : 0;
  mp.alpha = 0.01f;
  mp.beta = 0.5f;
  mp.hypotheses = 1024;
  mp.threshold = 1.0f;
  mp.refine = 3;
  mp.seed = 0;
  return ofdis_global_motion_fullres(s.ctx.get(), 0, b.n, b.n, &mp, b.frames.data() + b.hwc, b.fs, b.gm_models.data(),
                                     b.gm_stats.data(), b.gm_mask.data(), b.gm_res.data(), b.gm_reg.data(), b.w, b.h,
                                     OFDIS_MEM_HOST);
}

static int run_disparity(State& s, Batch& b) {
  const Options& o = s.o;
  const size_t np = (size_t)b.n * b.w * b.h;
  b.ddisp.resize(np);
  b.dstatus.resize(np);
  b.ddepth.resize(o.camera ? np : 0);
  b.dxyz.resize(o.camera ? 3 * np : 0);
  const int rc = ofdis_disparity_fullres(s.ctx.get(), 0, b.n, b.n, &o.dfilt, o.camera ? &o.dcam : nullptr,
                                         b.ddisp.data(), b.dstatus.data(), o.camera ? b.ddepth.data() : nullptr,
                                         o.camera ? b.dxyz.data() : nullptr, b.w, b.h, OFDIS_MEM_HOST);
  memset(b.dcount, 0, sizeof(b.dcount));
  for (size_t i = 0; i < np && rc == OFDIS_OK; ++i) {
    b.dcount[b.dstatus[i] < 5 ? b.dstatus[i] : 0] += 1;
    b.dcount[5] += b.dstatus[i] != 0 && !std::isnan(b.ddisp[i]);
  }
  return rc;
}

static void write_tracks(State& s, const ofdis_track_point* p, int count) {
  for (int i = 0; i < count; ++i)
    fprintf(s.out.tracks.f, "%d %d %d %.9g %.9g\n", s.tclip, s.tframe, p[i].id, (double)p[i].x, (double)p[i].y);
  ++s.tframe;
  ++s.tframes;
}

static void write_desc(State& s, int count) {
  const int tdim = s.o.tdim;
  for (int i = 0; i < count; ++i) {
    const ofdis_traj_record& r = s.trec[i];
    fprintf(s.out.desc.f, "%d %d %d %.9g %.9g %.9g %.9g %.9g", s.tclip, r.id, r.start, (double)r.mean_x,
            (double)r.mean_y, (double)r.sd_x, (double)r.sd_y, (double)r.length);
    const float* d = s.tdesc.data() + (size_t)i * tdim;
    for (int e = 0; e < tdim; ++e) fprintf(s.out.desc.f, " %.9g", (double)d[e]);
    fprintf(s.out.desc.f, "\n");
  }
}

// The tracked clip's end: --fisher takes its vector; the tracker's (and the descriptor stage's) counters go to the
// totals
static int end_track_clip(State& s) {
  ofdis_ctx* ctx = s.ctx.get();
  const ofdis_fisher_codebook& cb = s.o.fbook.cb;
  if (s.out.fisher.f) {
    ofdis_fisher_stats fs;
    const int rc = ofdis_fisher_take(ctx, s.fvec.data(), nullptr, &fs, OFDIS_MEM_HOST);
    if (rc != OFDIS_OK) return rc;
    fprintf(s.out.fisher.f, "%d %lld", s.tclip, fs.pushed);
    for (int b = 0; b < cb.nblocks; ++b) fprintf(s.out.fisher.f, " %lld", fs.n[b]);
    for (float v : s.fvec) fprintf(s.out.fisher.f, " %.9g", (double)v);
    fprintf(s.out.fisher.f, "\n");
    ++s.fclips;
    s.fpushed += fs.pushed;
    for (int b = 0; b < cb.nblocks; ++b) s.fskipped[b] += fs.skipped[b];
  }
  ofdis_track_stats st;
  if (ofdis_track_stats_get(ctx, &st) != OFDIS_OK) return OFDIS_OK;
  s.ttotal.seeded += st.seeded;
  s.ttotal.ended_leaves += st.ended_leaves;
  s.ttotal.ended_inconsistent += st.ended_inconsistent;
  s.ttotal.ended_boundary += st.ended_boundary;
  s.ttotal.dropped += st.dropped;
  ofdis_traj_stats ds;
  if (!s.o.traj_stage || ofdis_traj_stats_get(ctx, &ds) != OFDIS_OK) return OFDIS_OK;
  s.dtotal.emitted += ds.emitted;
  s.dtotal.rejected_static += ds.rejected_static;
  s.dtotal.rejected_erratic += ds.rejected_erratic;
  s.dtotal.rejected_jump += ds.rejected_jump;
  s.dtotal.rejected_camera += ds.rejected_camera;
  return OFDIS_OK;
}

// --tracks, with --descriptors / --fisher through the descriptor stage: a run that begins a clip begins the tracker on
// its first image1 (and the Fisher encoder), every run advances it through its image2 frames, and a run that ends the
// clip ends it
static int run_tracks(State& s, Batch& b) {
  const Options& o = s.o;
  ofdis_ctx* ctx = s.ctx.get();
  const int n = b.n, w = b.w, h = b.h;
  const double* models = o.gm_model ? b.gm_models.data() : nullptr;
  ofdis_track_params tp;
  tp.spacing = 8;
  tp.capacity = 4 * ((w + 7) / 8) * ((h + 7) / 8);
  tp.alpha = s.nop == 2 ? 0.01f : 0.0f;
  tp.beta = s.nop == 2 ? 0.5f : 1.0f;
  tp.mb_alpha = 0.01f;
  tp.mb_beta = 0.002f;
  tp.min_eig = 25.0f;
  s.tpoints.resize((size_t)n * tp.capacity);
  s.tcounts.resize(n);
  int rc = OFDIS_OK;
  for (const ClipRun& r : clip_runs(s.clips, b.j0, n)) {
    const int k0 = r.k0, k1 = r.k1;
    const uint8_t* im1 = b.frames.data() + (size_t)k0 * b.fs;
    const uint8_t* im2 = im1 + b.hwc;
    if (r.starts) {
      ++s.tclip;
      s.tframe = 0;
      rc = o.traj_stage ? ofdis_traj_begin(ctx, &tp, &o.trp, im1, s.tpoints.data(), s.tcounts.data(), w, h,
                                           OFDIS_MEM_HOST)
                        : ofdis_track_begin(ctx, &tp, im1, s.tpoints.data(), s.tcounts.data(), w, h, OFDIS_MEM_HOST);
      if (rc == OFDIS_OK && s.out.fisher.f) rc = ofdis_fisher_begin(ctx, &o.fbook.cb);
      if (rc == OFDIS_OK) write_tracks(s, s.tpoints.data(), s.tcounts[0]);
    }
    s.tndesc.resize(k1 - k0);
    if (rc == OFDIS_OK && o.traj_stage && !o.desc) {  // --fisher alone: the descriptors stay on the device
      rc = ofdis_traj_advance_fisher(ctx, k0, k1, n + k0, im2, b.fs, models ? models + (size_t)9 * k0 : nullptr,
                                     s.tpoints.data(), s.tcounts.data(), s.tndesc.data(), w, h, OFDIS_MEM_HOST);
    } else if (rc == OFDIS_OK && o.desc) {
      const size_t bound = (size_t)tp.capacity * ((k1 - k0 + 2 * o.trp.L - 2) / o.trp.L);
      s.trec.resize(bound);
      s.tdesc.resize(bound * o.tdim);
      rc = ofdis_traj_advance(ctx, k0, k1, n + k0, im2, b.fs, models ? models + (size_t)9 * k0 : nullptr,
                              s.tpoints.data(), s.tcounts.data(), s.trec.data(), s.tdesc.data(), s.tndesc.data(), w, h,
                              OFDIS_MEM_HOST);
      int total = 0;
      for (int k = 0; k < k1 - k0 && rc == OFDIS_OK; ++k) total += s.tndesc[k];
      if (rc == OFDIS_OK) write_desc(s, total);
      if (rc == OFDIS_OK && s.out.fisher.f) rc = ofdis_fisher_push(ctx, s.tdesc.data(), total, OFDIS_MEM_HOST);
    } else if (rc == OFDIS_OK) {
      rc = ofdis_track_advance(ctx, k0, k1, n + k0, im2, b.fs, s.tpoints.data(), s.tcounts.data(), w, h,
                               OFDIS_MEM_HOST);
    }
    for (int k = 0; k < k1 - k0 && rc == OFDIS_OK; ++k)
      write_tracks(s, s.tpoints.data() + (size_t)k * tp.capacity, s.tcounts[k]);
    if (rc == OFDIS_OK && r.ends) rc = end_track_clip(s);
    if (rc != OFDIS_OK) break;
  }
  return rc;
}

// --stabilize: `count` emitted frames of the clip being stabilised to DIR/stab_<clip>_<frame>.png and stab.txt
static void write_stab(State& s, const Batch& b, int count) {
  for (int i = 0; i < count; ++i) {
    const ofdis_stab_frame& f = s.sinfo[i];
    fprintf(s.out.stab.f, "%d %lld", s.sclip, f.frame);
    for (int e = 0; e < 9; ++e) fprintf(s.out.stab.f, " %.17g", f.correction[e]);
    fprintf(s.out.stab.f, " %.17g %d\n", f.lambda, f.status);
    char name[64];
    snprintf(name, sizeof(name), "/stab_%04d_%06lld.png", s.sclip, f.frame);
    save_png(as_rgb(s.sbuf.data() + (size_t)i * b.hwc, b.hwc, s.nochannels, s.png), b.w, b.h, s.nochannels, 8,
             (string(s.o.stab[2]) + name).c_str());
  }
}

// --stabilize: a run that begins a clip begins the stabiliser on its first image1, every run pushes its image2 frames
// with their --global-motion models, and a run that ends the clip emits the rest
static int run_stabilize(State& s, Batch& b) {
  ofdis_ctx* ctx = s.ctx.get();
  int rc = OFDIS_OK;
  for (const ClipRun& r : clip_runs(s.clips, b.j0, b.n)) {
    const uint8_t* im1 = b.frames.data() + (size_t)r.k0 * b.fs;
    if (r.starts) {
      rc = ofdis_stab_begin(ctx, &s.o.stp, s.o.stab_wts.data(), im1, b.w, b.h, OFDIS_MEM_HOST);
      if (rc != OFDIS_OK) break;
      ++s.sclip;
    }
    s.sbuf.resize((size_t)(r.k1 - r.k0) * b.hwc);
    s.sinfo.resize(r.k1 - r.k0);
    int count = 0;
    rc = ofdis_stab_push(ctx, r.k1 - r.k0, b.gm_models.data() + (size_t)9 * r.k0, im1 + b.hwc, b.fs, s.sbuf.data(),
                         s.sinfo.data(), &count, OFDIS_MEM_HOST);
    if (rc == OFDIS_OK) write_stab(s, b, count);
    if (rc == OFDIS_OK && r.ends) {
      s.sbuf.resize((size_t)s.o.stp.radius * b.hwc);
      s.sinfo.resize(s.o.stp.radius);
      rc = ofdis_stab_finish(ctx, s.sbuf.data(), s.sinfo.data(), &count, OFDIS_MEM_HOST);
      if (rc == OFDIS_OK) write_stab(s, b, count);
    }
    if (rc != OFDIS_OK) break;
  }
  return rc;
}

// A host-side failure whose refusal is printed already (every OFDIS_* status is <= 0)
static const int kRefused = 1;

// --gt: the forward slots against the batch's ground truth
static int run_eval(State& s, Batch& b) {
  const int n = b.n, w = b.w, h = b.h, nop = s.nop, nclasses = s.nclasses;
  s.gt_batch.resize((size_t)n * w * h * nop);
  for (int k = 0; k < n; ++k) {
    string err;
    const string& gt = s.in.gts[b.j0 + k];
    if (!read_gt_file(gt.c_str(), w, h, nop, s.gt_one, err)) return refuse(kRefused, "%s: %s", gt.c_str(), err.c_str());
    memcpy(s.gt_batch.data() + (size_t)k * w * h * nop, s.gt_one.data(), sizeof(float) * s.gt_one.size());
  }
  s.eval_pairs.resize((size_t)n * nclasses);
  const int rc = ofdis_flow_error_fullres(s.ctx.get(), 0, n, s.gt_batch.data(), s.o.bidir ? b.masks.data() : nullptr,
                                          nclasses, s.eval_pairs.data(), nullptr, w, h, OFDIS_MEM_HOST);
  for (int k = 0; k < n && rc == OFDIS_OK; ++k)
    for (int c = 0; c < nclasses; ++c) {
      add_stats(s.eval_total[0], s.eval_pairs[(size_t)k * nclasses + c]);
      if (s.o.bidir) add_stats(s.eval_total[1 + c], s.eval_pairs[(size_t)k * nclasses + c]);
    }
  return rc;
}

// --scene-flow: the pairs' disparities in, the scene flow and its evaluation, <stem>_disp1 and <stem>_sceneflow.pfm out
static int run_scene_flow(State& s, Batch& b) {
  const Options& o = s.o;
  const int n = b.n, w = b.w, h = b.h, nclasses = s.nclasses;
  const size_t pix = (size_t)w * h, j0 = b.j0;
  // positive disparities: the readers return this library's stereo convention, -d
  auto load = [&](const string& path, int fnop, float sign, float* dst) {
    string err;
    if (!read_gt_file(path.c_str(), w, h, fnop, s.gt_one, err)) {
      refuse(kRefused, "%s: %s", path.c_str(), err.c_str());
      return false;
    }
    for (size_t i = 0; i < s.gt_one.size(); ++i) dst[i] = sign * s.gt_one[i];
    return true;
  };
  const vector<string>& df = s.in.sf_files;
  const vector<string>& gf = s.in.sf_gts;
  b.sf_d0.resize(n * pix);
  b.sf_d1.resize(n * pix);
  b.sf_w.resize(n * pix);
  b.sf_m.resize(o.camera ? 3 * n * pix : 0);
  bool ok = true;
  for (int k = 0; k < n && ok; ++k)
    ok = load(df[2 * (j0 + k)], 1, -1.0f, &b.sf_d0[k * pix]) && load(df[2 * (j0 + k) + 1], 1, -1.0f, &b.sf_d1[k * pix]);
  if (o.sf_gtlist) {
    s.sf_g0.resize(n * pix);
    s.sf_g1.resize(n * pix);
    s.sf_gf.resize(2 * n * pix);
    for (int k = 0; k < n && ok; ++k)
      ok = load(gf[3 * (j0 + k)], 1, -1.0f, &s.sf_g0[k * pix]) && load(gf[3 * (j0 + k) + 1], 1, -1.0f, &s.sf_g1[k * pix]) &&
           load(gf[3 * (j0 + k) + 2], 2, 1.0f, &s.sf_gf[2 * k * pix]);
    s.sf_pairs.resize((size_t)n * nclasses);
  }
  if (!ok) return kRefused;
  const ofdis_sf_gt sgt{s.sf_g0.data(), s.sf_g1.data(), s.sf_gf.data()};
  const int rc = ofdis_scene_flow_fullres(s.ctx.get(), 0, n, b.sf_d0.data(), b.sf_d1.data(), pix, 1.0f,
                                          o.camera ? &o.dcam : nullptr, b.sf_w.data(), nullptr,
                                          o.camera ? b.sf_m.data() : nullptr, o.sf_gtlist ? &sgt : nullptr,
                                          o.bidir ? b.masks.data() : nullptr, nclasses,
                                          o.sf_gtlist ? s.sf_pairs.data() : nullptr, w, h, OFDIS_MEM_HOST);
  for (int k = 0; k < n && rc == OFDIS_OK && o.sf_gtlist; ++k) {
    ofdis_sf_stats all;
    memset(&all, 0, sizeof(all));
    for (int c = 0; c < nclasses; ++c) {
      add_sf_stats(all, s.sf_pairs[(size_t)k * nclasses + c]);
      add_sf_stats(s.sf_total[1 + c], s.sf_pairs[(size_t)k * nclasses + c]);
    }
    add_sf_stats(s.sf_total[0], all);
    if (s.verbosity > 0) print_sfeval(s.jobs[j0 + k].out.c_str(), 0, all);
  }
  for (int k = 0; k < n && rc == OFDIS_OK; ++k) {
    const string& out = s.jobs[j0 + k].out;
    if (o.kitti) save_kitti_disp(&b.sf_w[k * pix], w, h, with_suffix(out, "_disp1"));
    else save_pfm1(&b.sf_w[k * pix], w, h, with_suffix(out, "_disp1", ".pfm"));
    if (o.camera) save_pfm3(&b.sf_m[3 * k * pix], w, h, with_suffix(out, "_sceneflow", ".pfm").c_str());
  }
  return rc;
}

// --odometry: the rig's motion of every pair to odometry.txt, <stem>_objects.pgm and <stem>_objmotion.pfm; --gt-poses
// its error
static int run_odometry(State& s, Batch& b) {
  const int n = b.n, w = b.w, h = b.h;
  const size_t pix = (size_t)w * h;
  FILE* f = s.out.odo.f;
  ofdis_egomotion_params ep;
  memset(&ep, 0, sizeof(ep));
  ep.step = 8;
  ep.fb_check = s.o.bidir ? 1 : 0;
  ep.alpha = 0.01f;
  ep.beta = 0.5f;
  ep.edge_diff = 1.0f;
  ep.hypotheses = 1024;
  ep.threshold = 1.0f;
  ep.refine = 5;
  ep.seed = 0;
  b.odo_pose.resize((size_t)12 * n);
  s.odo_stats.resize(n);
  s.odo_mask.resize(n * pix);
  s.odo_om.resize(3 * n * pix);
  const int rc = ofdis_egomotion_fullres(s.ctx.get(), 0, n, n, &ep, b.sf_d0.data(), b.sf_d1.data(), pix, &s.o.dcam,
                                         b.odo_pose.data(), s.odo_stats.data(), s.odo_mask.data(), nullptr,
                                         s.odo_om.data(), w, h, OFDIS_MEM_HOST);
  for (int k = 0; k < n && rc == OFDIS_OK; ++k) {
    const int c = s.clips.clip[b.j0 + k], fr = s.clips.frame[b.j0 + k];
    const ofdis_motion_stats& st = s.odo_stats[k];
    const double* P = b.odo_pose.data() + (size_t)12 * k;
    const string& out = s.jobs[b.j0 + k].out;
    fprintf(f, "%d %d %d %d %d %d", c, fr, st.status, st.n_corr, st.ransac_inliers, st.n_inliers);
    for (int i = 0; i < 12; ++i) fprintf(f, " %.17g", P[i]);
    fprintf(f, "\n");
    s.odo_rel[c].insert(s.odo_rel[c].end(), P, P + 12);
    save_mask_pgm(s.odo_mask.data() + k * pix, w, h, with_suffix(out, "_objects", ".pgm").c_str());
    save_pfm3(&s.odo_om[3 * k * pix], w, h, with_suffix(out, "_objmotion", ".pfm").c_str());
    if (!s.o.odo_gtlist) continue;
    double te, re;
    const vector<double>& gt = s.in.odo_gt[c];
    pose_error(&gt[(size_t)12 * fr], &gt[(size_t)12 * (fr + 1)], P, &te, &re);
    s.odo_terr += te;
    s.odo_rerr += re;
    ++s.odo_eval;
    if (s.verbosity > 0) printf("ODOEVAL %d %d %.9g %.9g\n", c, fr, te, re);
  }
  return rc;
}

// The ground truth's relative motion of frames G0 -> G1 (camera-to-world): Q = inv(G1) G0, camera t to camera t+1
static void gt_relative(const double* G0, const double* G1, double* Q) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Q[4 * i + j] = G1[i] * G0[j] + G1[4 + i] * G0[4 + j] + G1[8 + i] * G0[8 + j];
    Q[4 * i + 3] = G1[i] * (G0[3] - G1[3]) + G1[4 + i] * (G0[7] - G1[7]) + G1[8 + i] * (G0[11] - G1[11]);
  }
}

// --mono-odometry: the camera's motion of every pair to monodometry.txt, <stem>_epimask.pgm and <stem>_depthrel.pfm;
// --gt-poses its rotation and translation-direction errors
static int run_mono(State& s, Batch& b) {
  const int n = b.n, w = b.w, h = b.h;
  const size_t pix = (size_t)w * h;
  FILE* f = s.out.mono.f;
  ofdis_relpose_params p = s.o.rpp;
  p.fb_check = s.o.bidir ? 1 : 0;
  s.mono_pose.resize((size_t)12 * n);
  s.mono_stats.resize(n);
  s.mono_mask.resize(n * pix);
  s.mono_depth.resize(n * pix);
  const int rc = ofdis_relpose_fullres(s.ctx.get(), 0, n, n, &p, s.mono_pose.data(), s.mono_stats.data(),
                                       s.mono_mask.data(), nullptr, s.mono_depth.data(), w, h, OFDIS_MEM_HOST);
  for (int k = 0; k < n && rc == OFDIS_OK; ++k) {
    const int c = s.clips.clip[b.j0 + k], fr = s.clips.frame[b.j0 + k];
    const ofdis_motion_stats& st = s.mono_stats[k];
    const double* P = s.mono_pose.data() + (size_t)12 * k;
    const string& out = s.jobs[b.j0 + k].out;
    fprintf(f, "%d %d %d", c, fr, st.status);
    for (int i = 0; i < 12; ++i) fprintf(f, " %.17g", P[i]);
    fprintf(f, "\n");
    s.mono_rel[c].insert(s.mono_rel[c].end(), P, P + 12);
    save_mask_pgm(s.mono_mask.data() + k * pix, w, h, with_suffix(out, "_epimask", ".pgm").c_str());
    save_pfm1(&s.mono_depth[k * pix], w, h, with_suffix(out, "_depthrel", ".pfm"));  // as _depth.pfm
    if (!s.o.odo_gtlist || st.status != 0) continue;
    const vector<double>& gt = s.in.odo_gt[c];
    double Q[12];
    gt_relative(&gt[(size_t)12 * fr], &gt[(size_t)12 * (fr + 1)], Q);
    double tr = 0.0, dt = 0.0, nq = 0.0, np_ = 0.0;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) tr += Q[4 * i + j] * P[4 * i + j];
      dt += Q[4 * i + 3] * P[4 * i + 3];
      nq += Q[4 * i + 3] * Q[4 * i + 3];
      np_ += P[4 * i + 3] * P[4 * i + 3];
    }
    const double kDeg = 180.0 / 3.14159265358979323846;
    const double re = acos(std::min(1.0, std::max(-1.0, 0.5 * (tr - 1.0)))) * kDeg;
    const double te = acos(std::min(1.0, std::max(-1.0, dt / sqrt(nq * np_)))) * kDeg;
    s.mono_rerr += re;
    s.mono_terr += te;
    ++s.mono_eval;
    if (s.verbosity > 0) printf("MONOEVAL %d %d %.9g %.9g\n", c, fr, re, te);
  }
  return rc;
}

// --fuse: the end of a clip's volume, pushed with its last image2: the surface to DIR/fused_<clip>.ply, with --mesh
// the triangle mesh to DIR/fused_<clip>_mesh.ply
static int end_fuse_clip(State& s, const Batch& b, const ClipRun& r) {
  ofdis_ctx* ctx = s.ctx.get();
  const int c = s.clips.clip[b.j0 + r.k0], w = b.w, h = b.h;
  const size_t pix = (size_t)w * h;
  int rc = ofdis_fuse_push(ctx, 1, &b.sf_d1[(r.k1 - 1) * pix], pix, &s.fuse_poses[(size_t)12 * (r.k1 - r.k0)],
                           &s.o.dcam, INFINITY, b.frames.data() + (size_t)(r.k1 - 1) * b.fs + b.hwc, b.fs, w, h,
                           OFDIS_MEM_HOST);
  ++s.fuse_frames;
  long count = 0;
  if (rc == OFDIS_OK) rc = ofdis_fuse_extract(ctx, 1.0f, nullptr, 0, &count, OFDIS_MEM_HOST);
  if (rc != OFDIS_OK) return rc;
  s.fuse_pts.resize(count);
  rc = ofdis_fuse_extract(ctx, 1.0f, s.fuse_pts.data(), count, &count, OFDIS_MEM_HOST);
  if (rc != OFDIS_OK) return rc;
  char name[32];
  snprintf(name, sizeof(name), "/fused_%04d.ply", c);
  string path = string(s.o.odo_dir) + name;
  if (!write_fused_ply(path, s.fuse_pts.data(), count, s.nochannels, false, nullptr, 0))
    return refuse(kRefused, "cannot write %s", path.c_str());
  if (s.verbosity > 0) printf("FUSE clip %d frames %d points %ld\n", c, s.fuse_frames, count);
  if (!s.o.mesh) return OFDIS_OK;
  // the mesh's vertices are the points just extracted: only the faces come back
  long nv = 0, nf = 0;
  rc = ofdis_fuse_mesh(ctx, 1.0f, nullptr, 0, &nv, nullptr, 0, &nf, OFDIS_MEM_HOST);
  if (rc != OFDIS_OK) return rc;
  s.fuse_faces.resize((size_t)3 * nf);
  rc = ofdis_fuse_mesh(ctx, 1.0f, nullptr, 0, &nv, s.fuse_faces.data(), nf, &nf, OFDIS_MEM_HOST);
  if (rc != OFDIS_OK) return rc;
  snprintf(name, sizeof(name), "/fused_%04d_mesh.ply", c);
  path = string(s.o.odo_dir) + name;
  if (!write_fused_ply(path, s.fuse_pts.data(), count, s.nochannels, true, s.fuse_faces.data(), nf))
    return refuse(kRefused, "cannot write %s", path.c_str());
  if (s.verbosity > 0) printf("MESH clip %d vertices %ld faces %ld\n", c, nv, nf);
  return OFDIS_OK;
}

// --fuse: a run that begins a clip begins its volume; every run pushes its image1 disparities with their chained poses,
// and a run that ends the clip ends the volume
static int run_fuse(State& s, Batch& b) {
  static const double kIdentity[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  const size_t pix = (size_t)b.w * b.h;
  int rc = OFDIS_OK;
  for (const ClipRun& r : clip_runs(s.clips, b.j0, b.n)) {
    if (r.starts) {
      memcpy(s.fuse_T, kIdentity, sizeof(s.fuse_T));
      s.fuse_frames = 0;
      rc = ofdis_fuse_begin(s.ctx.get(), &s.o.fuse_p);
      if (rc != OFDIS_OK) break;
    }
    s.fuse_poses.resize((size_t)12 * (r.k1 - r.k0 + 1));
    for (int k = r.k0; k < r.k1; ++k) {
      memcpy(&s.fuse_poses[(size_t)12 * (k - r.k0)], s.fuse_T, sizeof(s.fuse_T));
      chain_pose(s.fuse_T, b.odo_pose.data() + (size_t)12 * k);
    }
    memcpy(&s.fuse_poses[(size_t)12 * (r.k1 - r.k0)], s.fuse_T, sizeof(s.fuse_T));
    rc = ofdis_fuse_push(s.ctx.get(), r.k1 - r.k0, &b.sf_d0[r.k0 * pix], pix, s.fuse_poses.data(), &s.o.dcam, INFINITY,
                         b.frames.data() + (size_t)r.k0 * b.fs, b.fs, b.w, b.h, OFDIS_MEM_HOST);
    s.fuse_frames += r.k1 - r.k0;
    if (rc == OFDIS_OK && r.ends) rc = end_fuse_clip(s, b, r);
    if (rc != OFDIS_OK) break;
  }
  return rc;
}

// The device stages of a batch, in order; the first failure ends them
static int run_stages(State& s, Batch& b) {
  const Options& o = s.o;
  int rc = run_flows(s, b);
  if (rc == OFDIS_OK && o.interp_arg) rc = run_interpolate(s, b);
  if (rc == OFDIS_OK && o.conf_arg) rc = run_confidence(s, b);
  if (rc == OFDIS_OK && o.gm_model) rc = run_global_motion(s, b);
  if (rc == OFDIS_OK && o.disp_on) rc = run_disparity(s, b);
  if (rc == OFDIS_OK && o.tracks) rc = run_tracks(s, b);
  if (rc == OFDIS_OK && o.stab[0]) rc = run_stabilize(s, b);
  if (rc == OFDIS_OK) rc = ofdis_sync(s.ctx.get());
  if (rc == OFDIS_OK && o.gtlist) rc = run_eval(s, b);
  if (rc == OFDIS_OK && o.sf_list) rc = run_scene_flow(s, b);
  if (rc == OFDIS_OK && o.odo_dir) rc = run_odometry(s, b);
  if (rc == OFDIS_OK && o.mono_dir) rc = run_mono(s, b);
  if (rc == OFDIS_OK && o.fuse) rc = run_fuse(s, b);
  return rc;
}

// Every pair's <stem><ext> (KITTI's PNG with --kitti), with --bidirectional <stem>_bw<ext> and <stem>_occ.pgm
static void write_flows(State& s, const Batch& b) {
  const int w = b.w, h = b.h, nop = s.nop, kch = nop == 2 ? 3 : 1;
  ImageF img;
  img.w = w;
  img.h = h;
  img.c = nop;
  auto save = [&](int slot, const string& path) {
    if (s.o.kitti) {
      save_png(b.kflows.data() + (size_t)slot * w * h * kch, w, h, kch, 16, path.c_str());
      return;
    }
    img.px.assign(b.flows.begin() + (size_t)slot * w * h * nop, b.flows.begin() + (size_t)(slot + 1) * w * h * nop);
    if (SELECTMODE == 1) SaveFlowFile(img, path.c_str());
    else SavePFMFile(img, path.c_str());
  };
  for (int k = 0; k < b.n; ++k) {
    const string& out = s.jobs[b.j0 + k].out;
    save(k, out);
    if (!s.o.bidir) continue;
    save(b.n + k, with_suffix(out, "_bw"));
    save_mask_pgm(b.masks.data() + (size_t)k * w * h, w, h, with_suffix(out, "_occ", ".pgm").c_str());
  }
}

// --global-motion: every pair's line, <stem>_residual<ext>, <stem>_moving.pgm and <stem>_registered.png
static void write_global_motion(State& s, const Batch& b) {
  const int w = b.w, h = b.h;
  for (int k = 0; k < b.n; ++k) {
    const string& o = s.jobs[b.j0 + k].out;
    fprintf(s.out.gm.f, "%s", with_suffix(o, "", "").c_str());
    for (int i = 0; i < 9; ++i) fprintf(s.out.gm.f, " %.17g", b.gm_models[(size_t)9 * k + i]);
    fprintf(s.out.gm.f, " %d %d %d\n", b.gm_stats[k].status, b.gm_stats[k].n_corr, b.gm_stats[k].n_inliers);
    const float* r = b.gm_res.data() + (size_t)2 * k * w * h;
    if (s.o.kitti) {
      save_kitti_flow(r, w, h, with_suffix(o, "_residual"));
    } else {
      ImageF f;
      f.w = w;
      f.h = h;
      f.c = 2;
      f.px.assign(r, r + (size_t)2 * w * h);
      SaveFlowFile(f, with_suffix(o, "_residual").c_str());
    }
    save_mask_pgm(b.gm_mask.data() + (size_t)k * w * h, w, h, with_suffix(o, "_moving", ".pgm").c_str());
    save_png(as_rgb(b.gm_reg.data() + (size_t)k * b.hwc, b.hwc, s.nochannels, s.png), w, h, s.nochannels, 8,
             with_suffix(o, "_registered", ".png").c_str());
  }
}

// The filtered disparities: every pair's <stem>_filtered<ext>, with --camera <stem>_depth.pfm and <stem>.ply
static void write_disparities(State& s, const Batch& b) {
  const int w = b.w, h = b.h, ch = s.nochannels;
  vector<uint8_t> ply;
  for (int k = 0; k < b.n; ++k) {
    const size_t o = (size_t)k * w * h;
    const string& out = s.jobs[b.j0 + k].out;
    if (s.o.kitti) save_kitti_disp(&b.ddisp[o], w, h, with_suffix(out, "_filtered"));
    else save_pfm1(&b.ddisp[o], w, h, with_suffix(out, "_filtered"));  // the sign of <stem><ext>
    if (!s.o.camera) continue;
    save_pfm1(&b.ddepth[o], w, h, with_suffix(out, "_depth", ".pfm"));
    const uint8_t* im1 = b.frames.data() + (size_t)k * b.fs;
    size_t npts = 0;
    ply.clear();
    for (size_t i = 0; i < (size_t)w * h; ++i) {
      if (!std::isfinite(b.ddepth[o + i])) continue;
      const uint8_t* qb = reinterpret_cast<const uint8_t*>(b.dxyz.data() + (o + i) * 3);
      const uint8_t* c = im1 + i * ch;
      const uint8_t rgb[3] = {ch == 3 ? c[2] : c[0], c[ch == 3 ? 1 : 0], c[0]};  // the decoder's BGR
      ply.insert(ply.end(), qb, qb + 12);
      ply.insert(ply.end(), rgb, rgb + 3);
      ++npts;
    }
    FILE* pf = fopen(with_suffix(out, "", ".ply").c_str(), "wb");
    if (!pf) {
      cout << "WriteFile: could not open file" << endl;
      continue;
    }
    fprintf(pf, "ply\nformat binary_little_endian 1.0\nelement vertex %zu\nproperty float x\nproperty float y\n"
                "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n", npts);
    if (fwrite(ply.data(), 1, ply.size(), pf) != ply.size()) cout << "WriteFile: problem writing data" << endl;
    fclose(pf);
  }
  if (s.verbosity > 0)
    printf("DISP pairs %d valid %zu inconsistent %zu leaves %zu range %zu speckle %zu filled %zu\n", b.n, b.dcount[0],
           b.dcount[1], b.dcount[2], b.dcount[3], b.dcount[4], b.dcount[5]);
}

// The batch's per-pair files (KITTI's PNGs first and the .flo / .pfm files last, as they have always gone)
static void write_outputs(State& s, const Batch& b) {
  const Options& o = s.o;
  const int w = b.w, h = b.h;
  if (o.kitti) write_flows(s, b);
  for (int k = 0; k < b.n && o.color; ++k) {
    const string& out = s.jobs[b.j0 + k].out;
    save_png(b.colors.data() + (size_t)k * w * h * 3, w, h, 3, 8, with_suffix(out, "_color", ".png").c_str());
    if (o.bidir)
      save_png(b.colors.data() + (size_t)(b.n + k) * w * h * 3, w, h, 3, 8, with_suffix(out, "_bw_color", ".png").c_str());
  }
  for (int k = 0; k < b.n && o.interp_arg; ++k)
    save_png(as_rgb(b.interp.data() + (size_t)k * b.hwc, b.hwc, s.nochannels, s.png), w, h, s.nochannels, 8,
             with_suffix(s.jobs[b.j0 + k].out, "_interp", ".png").c_str());
  if (o.gm_model) write_global_motion(s, b);
  if (o.disp_on) write_disparities(s, b);
  if (o.conf_arg) {
    double sum = 0.0;
    for (int k = 0; k < b.n; ++k)
      save_pfm1(b.conf.data() + (size_t)k * w * h, w, h, with_suffix(s.jobs[b.j0 + k].out, "_conf", ".pfm"));
    for (const float c : b.conf) sum += c;
    if (s.verbosity > 0) printf("CONF pairs %d mean %.9g\n", b.n, sum / (double)b.conf.size());
  }
  if (!o.kitti) write_flows(s, b);
}

// --odometry: every clip's camera-to-world poses to DIR/poses_<clip>.txt
// --mono-odometry: the same into its own DIR, each unit step scaled by the ground truth's step length with --gt-poses
static int write_poses(const State& s) {
  for (int mono = 0; mono < 2; ++mono) {
    const vector<vector<double>>& rel = mono ? s.mono_rel : s.odo_rel;
    for (size_t c = 0; c < rel.size(); ++c) {
      char name[32];
      snprintf(name, sizeof(name), "/poses_%04zu.txt", c);
      const string path = string(mono ? s.o.mono_dir : s.o.odo_dir) + name;
      FILE* f = fopen(path.c_str(), "w");
      double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
      for (size_t k = 0; f && k <= rel[c].size() / 12; ++k) {
        if (k > 0) {
          double P[12];
          memcpy(P, &rel[c][12 * (k - 1)], sizeof(P));
          if (mono && s.o.odo_gtlist) {
            const double* G0 = &s.in.odo_gt[c][12 * (k - 1)];
            const double* G1 = G0 + 12;
            const double dx = G1[3] - G0[3], dy = G1[7] - G0[7], dz = G1[11] - G0[11];
            const double len = sqrt(dx * dx + dy * dy + dz * dz);
            for (int i = 0; i < 3; ++i) P[4 * i + 3] *= len;
          }
          chain_pose(T, P);
        }
        for (int i = 0; i < 12; ++i) fprintf(f, i ? " %.17g" : "%.17g", T[i]);
        fprintf(f, "\n");
      }
      if (!f || fclose(f) != 0) return refuse(1, "cannot write %s", path.c_str());
    }
  }
  return 0;
}

static void print_summary(const State& s, timeval& tv) {
  if (s.verbosity <= 0) return;
  const Options& o = s.o;
  static const char* const kClassNames[3] = {"consistent", "inconsistent", "leaves"};
  printf("TIME (%zu pairs, load + flow + save) (ms): %3g\n", s.done, elapsed_ms(tv));
  if (s.seq_pairs) printf("SEQUENCE (%zu of %zu pairs from %zu decoded frames)\n", s.seq_pairs, s.done, s.seq_decoded);
  if (o.warm) printf("WARM START (%zu of %zu pairs from the previous pair's flow)\n", s.warm_pairs, s.done);
  if (o.tracks)
    printf("TRACKS clips %d frames %zu seeded %lld leaves %lld inconsistent %lld boundary %lld dropped %lld\n",
           s.tclip + 1, s.tframes, s.ttotal.seeded, s.ttotal.ended_leaves, s.ttotal.ended_inconsistent,
           s.ttotal.ended_boundary, s.ttotal.dropped);
  if (o.desc)
    printf("DESCRIPTORS clips %d emitted %lld static %lld erratic %lld jump %lld camera %lld\n", s.tclip + 1,
           s.dtotal.emitted, s.dtotal.rejected_static, s.dtotal.rejected_erratic, s.dtotal.rejected_jump,
           s.dtotal.rejected_camera);
  if (o.fisher[0]) {
    printf("FISHER clips %d descriptors %lld skipped", s.fclips, s.fpushed);
    for (int b = 0; b < o.fbook.cb.nblocks; ++b) printf(" %lld", s.fskipped[b]);
    printf("\n");
  }
  if (o.gtlist) {
    print_eval("", s.done, s.eval_total[0]);
    for (int c = 0; c < s.nclasses && o.bidir; ++c) print_eval(kClassNames[c], s.done, s.eval_total[1 + c]);
  }
  if (o.odo_dir && o.odo_gtlist)
    printf("ODOEVAL (%zu pairs) t_err %.9g r_err %.9g\n", s.odo_eval, s.odo_eval ? s.odo_terr / s.odo_eval : 0.0,
           s.odo_eval ? s.odo_rerr / s.odo_eval : 0.0);
  if (o.mono_dir && o.odo_gtlist)
    printf("MONOEVAL (%zu pairs) r_err %.9g t_dir_err %.9g\n", s.mono_eval,
           s.mono_eval ? s.mono_rerr / s.mono_eval : 0.0, s.mono_eval ? s.mono_terr / s.mono_eval : 0.0);
  if (o.sf_gtlist) {
    print_sfeval("", s.done, s.sf_total[0]);
    for (int c = 0; c < s.nclasses && o.bidir; ++c) print_sfeval(kClassNames[c], s.done, s.sf_total[1 + c]);
  }
}

int main(int argc, char** argv) {
  if (argc < 2) {
    fprintf(stderr,
            "usage: %s listfile [--batch N | --warm-start] [--bidirectional] [--gt gtlist] [--kitti]\n"
            "       [--color [--color-max M]] [--interpolate T]\n"
            "       [--tracks PATH [--descriptors PATH] [--fisher CODEBOOK PATH]]\n"
            "       [--lr-check] [--speckle N R] [--fill] [--camera fx,fy,cx,cy,baseline,doffs]\n"
            "       [--global-motion similarity|affine|homography PATH [--stabilize RADIUS CROP DIR]]\n"
            "       [--scene-flow DISPLIST [--gt-scene-flow GTLIST]]\n"
            "       [--odometry DIR [--gt-poses LIST] [--fuse voxel,trunc,x0,y0,z0,nx,ny,nz [--mesh]]]\n"
            "       [oppoint | 20 parameters (README.md:66-88)]\n"
            "  --warm-start: latency mode for video, one pair per launch; a pair whose image1 is the previous pair's\n"
            "  image2 starts from that pair's flow (the reference's init flow); a clip then runs serially\n"
            "  --bidirectional: also the backward flow (stereo: the right view's disparity) of every pair, written to\n"
            "  <stem>_bw<ext>, and the forward-backward consistency mask to <stem>_occ.pgm (0 consistent,\n"
            "  255 inconsistent, 128 leaves the frame); not with --warm-start\n"
            "  --gt gtlist: ground-truth files (.flo / .pfm, or KITTI's 16-bit PNG), one per pair in list order; prints\n"
            "  EVAL lines (end-point error, shares above 1, 3, 5 px, KITTI outliers; with --bidirectional also per\n"
            "  consistency class)\n"
            "  --kitti: write every flow (and _bw) output as KITTI's 16-bit PNG (flow RGB16, stereo gray16 disparity),\n"
            "  whatever its extension\n"
            "  --color: also write <stem>_color.png (and <stem>_bw_color.png), the 8-bit RGB color coding of every\n"
            "  output (flow: Middlebury's color wheel, stereo: KITTI's disparity colors), colored on the device\n"
            "  --color-max M: color every pair with the scale M (a positive finite number) instead of its own maximum\n"
            "  --interpolate T: also write <stem>_interp.png, the frame at time T (0 < T < 1) between image1 and image2,\n"
            "  synthesised on the device from the forward and backward flows; not with --warm-start\n"
            "  --tracks PATH: dense point trajectories through every clip of the list, written to PATH as lines\n"
            "  `clip frame id x y`; not with --warm-start\n"
            "  --descriptors PATH: flow only, with --tracks; the trajectory descriptors (shape, HOG, HOF, MBH) of every\n"
            "  15-frame segment of the tracks, camera-compensated with the --global-motion models when given, written to\n"
            "  PATH as lines `clip id start mean_x mean_y sd_x sd_y length` and 426 floats; frames of at least 32 x 32;\n"
            "  not with --warm-start\n"
            "  --fisher CODEBOOK PATH: flow only, with --tracks; one Fisher vector per clip of the descriptors above,\n"
            "  encoded on the device with the codebook file CODEBOOK (python -m of_dis_b200.fisher_fit), written to\n"
            "  PATH as lines `clip n_desc n_0 .. n_4` and the vector; not with --warm-start\n"
            "  --lr-check, --speckle N R, --fill, --camera ...: stereo only; also write <stem>_filtered<ext>, the\n"
            "  disparity without the pixels that fail the left-right check and the speckles of at most N pixels (R px),\n"
            "  holes filled with the background disparity, and with --camera <stem>_depth.pfm and <stem>.ply;\n"
            "  not with --warm-start\n"
            "  --global-motion MODEL PATH: flow only; the camera motion of every pair, one line per pair in PATH, and\n"
            "  <stem>_residual<ext>, <stem>_moving.pgm and <stem>_registered.png; not with --warm-start\n"
            "  --stabilize RADIUS CROP DIR: flow only, with --global-motion; every clip stabilised along its smoothed\n"
            "  camera path (RADIUS 1..64 frames each side, CROP 0 <= CROP < 0.5 cut from each side), written to\n"
            "  DIR/stab_<clip>_<frame>.png, the corrections to DIR/stab.txt; not with --warm-start\n"
            "  --scene-flow DISPLIST (flow binaries): the disparities of image1 and image2 of every pair (PFM or KITTI\n"
            "  PNG) give <stem>_disp1.pfm (<stem>_disp1<ext> with --kitti), and with --camera <stem>_sceneflow.pfm;\n"
            "  --gt-scene-flow GTLIST: disp0, disp1 and flow ground truth per pair, SFEVAL lines; not with --warm-start\n"
            "  --odometry DIR (flow binaries, with --scene-flow and --camera): the rig's ego-motion of every pair to\n"
            "  DIR/odometry.txt, each clip's KITTI poses to DIR/poses_<clip>.txt, <stem>_objects.pgm and\n"
            "  <stem>_objmotion.pfm; --gt-poses LIST: one KITTI poses file per clip, ODOEVAL lines; not with --warm-start\n"
            "  --fuse voxel,trunc,x0,y0,z0,nx,ny,nz (flow binaries, with --odometry): every clip's disparities fused\n"
            "  into a TSDF volume of nx x ny x nz voxels from (x0, y0, z0), its surface points to DIR/fused_<clip>.ply;\n"
            "  not with --warm-start\n"
            "  --mesh (with --fuse): also the volume's triangle mesh to DIR/fused_<clip>_mesh.ply\n",
            argv[0]);
    return 2;
  }
  Options o;
  if (int rc = parse_flags(argc, argv, o)) return rc;
  if (int rc = check_options(o)) return rc;
  vector<string> words;
  if (!read_words(argv[1], words)) return refuse(1, "cannot read %s", argv[1]);
  vector<Job> jobs;
  for (size_t i = 0; i + 3 <= words.size(); i += 3) jobs.push_back({words[i], words[i + 1], words[i + 2]});
  const ClipIndex clips = index_clips(jobs);
  Inputs in;
  if (int rc = read_inputs(o, jobs, clips, in)) return rc;
  ListOutputs out;
  if (int rc = open_outputs(o, jobs, out)) return rc;
  timeval tv;
  gettimeofday(&tv, NULL);
  State s(o, jobs, clips, in, out);
  Batch b;
  for (size_t j0 = 0; j0 < jobs.size(); j0 += b.n) {
    if (int rc = load_batch(s, b, j0)) return rc;
    CliParams P;
    parse_cli_params(o.nnum, o.nums, b.w, P);
    s.verbosity = P.verbosity;
    if (int rc = ensure_context(s, b, P)) return rc;
    const int rc = run_stages(s, b);
    if (rc == kRefused) return 1;
    if (rc != OFDIS_OK) return refuse(1, "%s", ofdis_last_error(s.ctx.get()));
    write_outputs(s, b);
    s.done += b.n;
  }
  s.ctx.reset();
  if (int rc = out.close()) return rc;
  if (int rc = write_poses(s)) return rc;
  print_summary(s, tv);
  return 0;
}
#else
int main(int argc, char** argv) {
  timeval tv;
  gettimeofday(&tv, NULL);
  if (argc < 4) {
    fprintf(stderr,
            "usage: %s image1 image2 outputfile [oppoint | 20 parameters (README.md:66-88) [hasinfile [infile]]]\n"
            "  hasinfile 1: start from the flow in infile (.flo for flow, .pfm for stereo, the size of the images);\n"
            "  the images are then padded to multiples of 2^(lv_f+1) (run_dense.cpp:292-301)\n", argv[0]);
    return 2;
  }
  if (argc > 5 && (argc < 24 || argc > 26)) {
    fprintf(stderr, "error: expected 0, 1 or exactly 20 numbers (+ hasinfile [infile]) after the three paths, got %d\n",
            argc - 4);
    return 2;
  }
  const bool hasinfile = argc >= 25 && atoi(argv[24]) != 0;
  if (argc >= 25 && (hasinfile ? argc != 26 : argc != 25)) {
    fprintf(stderr, "error: hasinfile 1 takes exactly one infile, hasinfile 0 none\n");
    return 2;
  }
  const char* infile = hasinfile ? argv[25] : nullptr;
  const char *imgfile_ao = argv[1], *imgfile_bo = argv[2], *outfile = argv[3];
  const int nochannels = (SELECTCHANNEL == 3) ? 3 : 1;
  const int nop = (SELECTMODE == 1) ? 2 : 1;
  Image8 a8, b8;
  if (!load_image(imgfile_ao, nochannels, a8) || !load_image(imgfile_bo, nochannels, b8)) {
    fprintf(stderr, "error: cannot read input images (supported: binary PGM/PPM, 8-bit non-interlaced PNG)\n");
    return 1;
  }
  if (a8.w != b8.w || a8.h != b8.h) {
    fprintf(stderr, "error: image sizes differ\n");
    return 1;
  }
  const int width_org = a8.w, height_org = a8.h;

  // *** parameters (run_dense.cpp:219-294)
  CliParams P;
  parse_cli_params(argc > 5 ? 20 : argc - 4, argv + 4, width_org, P);
  // the init flow (run_dense.cpp:355-378), read and checked before any device work
  vector<float> initflow_org;
  if (hasinfile) {
    string err;
    if (!read_flow_file(infile, width_org, height_org, (SELECTMODE == 1) ? 2 : 1, "init-flow file", initflow_org, err)) {
      fprintf(stderr, "error: %s: %s\n", infile, err.c_str());
      return 1;
    }
  }
  const int lv_f = P.lv_f, lv_l = P.lv_l, maxiter = P.maxiter, miniter = P.miniter, patchsz = P.patchsz,
            patnorm = P.patnorm, costfct = P.costfct, tv_innerit = P.tv_innerit, tv_solverit = P.tv_solverit,
            verbosity = P.verbosity;
  const float mindprate = P.mindprate, mindrrate = P.mindrrate, minimgerr = P.minimgerr, poverl = P.poverl,
              tv_alpha = P.tv_alpha, tv_gamma = P.tv_gamma, tv_delta = P.tv_delta, tv_sor = P.tv_sor;
  const bool usefbcon = P.usefbcon, usetvref = P.usetvref;

  // *** pad so that width/height are divisible by 2^lv_f, or 2^(lv_f+1) with an init flow (run_dense.cpp:298-311)
  int padw = 0, padh = 0;
  const int scfct = (int)pow(2, hasinfile ? lv_f + 1 : lv_f);
  int div = width_org % scfct;
  if (div > 0) padw = scfct - div;
  div = height_org % scfct;
  if (div > 0) padh = scfct - div;
  auto to_float = [&](const Image8& s) {
    ImageF f;
    f.w = s.w; f.h = s.h; f.c = s.c;
    f.px.resize(s.px.size());
    for (size_t i = 0; i < s.px.size(); ++i) f.px[i] = (float)s.px[i];
    return pad(f, (int)floor((float)padh / 2.0f), (int)ceil((float)padh / 2.0f), (int)floor((float)padw / 2.0f),
               (int)ceil((float)padw / 2.0f), true);
  };
  // Default: pyramid, gradients, paddings, upsampling and crop run on the device, bit-identical to
  // the host restatement below (tests/test_gpu_parity.py); OFDIS_HOST_PYRAMID=1 keeps them on the
  // host and hands OFClass the float pyramids exactly like run_dense.cpp:391-400.
  const char* hp = getenv("OFDIS_HOST_PYRAMID");
  if (!(hp && atoi(hp))) {
    if (verbosity > 1) printf("TIME (Image loading     ) (ms): %3g\n", elapsed_ms(tv));
    ImageF out;
    out.w = width_org;
    out.h = height_org;
    out.c = nop;
    out.px.assign((size_t)out.w * out.h * nop, 0.f);
    if (verbosity > 1) printf("TIME (Pyramide+Gradients) (ms): %3g\n", elapsed_ms(tv));  // inside the run below
    try {
      OFC::OFClass ofc(a8.px.data(), b8.px.data(), width_org, height_org, out.px.data(), nullptr, lv_f, lv_l, maxiter,
                       miniter, mindprate, mindrrate, minimgerr, patchsz, poverl, usefbcon, costfct, nochannels,
                       patnorm, usetvref, tv_alpha, tv_gamma, tv_delta, tv_innerit, tv_solverit, tv_sor, verbosity, nop,
                       0, hasinfile ? initflow_org.data() : nullptr);
    } catch (const std::exception& e) {
      fprintf(stderr, "error: %s\n", e.what());
      return 1;
    }
    if (verbosity > 1) gettimeofday(&tv, NULL);
    if (SELECTMODE == 1) SaveFlowFile(out, outfile);
    else SavePFMFile(out, outfile);
    if (verbosity > 1) printf("TIME (Saving flow file  ) (ms): %3g\n", elapsed_ms(tv));
    return 0;
  }
  ImageF img_ao_fmat = to_float(a8), img_bo_fmat = to_float(b8);
  const int szw = img_ao_fmat.w, szh = img_ao_fmat.h;
  if (verbosity > 1) printf("TIME (Image loading     ) (ms): %3g\n", elapsed_ms(tv));

  // *** pyramids (run_dense.cpp:325-344)
  vector<const float*> img_ao_pyr(lv_f + 1), img_bo_pyr(lv_f + 1), img_ao_dx_pyr(lv_f + 1), img_ao_dy_pyr(lv_f + 1),
      img_bo_dx_pyr(lv_f + 1), img_bo_dy_pyr(lv_f + 1);
  vector<ImageF> pa, pax, pay, pb, pbx, pby;
  ConstructImgPyramide(img_ao_fmat, pa, pax, pay, img_ao_pyr.data(), img_ao_dx_pyr.data(), img_ao_dy_pyr.data(), lv_f, patchsz);
  ConstructImgPyramide(img_bo_fmat, pb, pbx, pby, img_bo_pyr.data(), img_bo_dx_pyr.data(), img_bo_dy_pyr.data(), lv_f, patchsz);
  if (verbosity > 1) printf("TIME (Pyramide+Gradients) (ms): %3g\n", elapsed_ms(tv));

  // *** init flow: replicate padding, x 2^-(lv_f+1), INTER_AREA to level lv_f+1 (run_dense.cpp:355-378)
  ImageF initflow;
  if (hasinfile) {
    ImageF fl;
    fl.w = width_org; fl.h = height_org; fl.c = nop;
    fl.px = initflow_org;
    initflow = initflow_level(pad(fl, (int)floor((float)padh / 2.0f), (int)ceil((float)padh / 2.0f),
                                  (int)floor((float)padw / 2.0f), (int)ceil((float)padw / 2.0f), true), lv_f);
  }

  // *** main algorithm (run_dense.cpp:383-400)
  const int sc_fct = (int)pow(2, lv_l);
  ImageF flowout;
  flowout.w = szw / sc_fct;
  flowout.h = szh / sc_fct;
  flowout.c = nop;
  flowout.px.assign((size_t)flowout.w * flowout.h * nop, 0.f);
  try {
    OFC::OFClass ofc(img_ao_pyr.data(), img_ao_dx_pyr.data(), img_ao_dy_pyr.data(), img_bo_pyr.data(),
                     img_bo_dx_pyr.data(), img_bo_dy_pyr.data(), patchsz, flowout.px.data(),
                     hasinfile ? initflow.px.data() : nullptr, szw, szh, lv_f,
                     lv_l, maxiter, miniter, mindprate, mindrrate, minimgerr, patchsz, poverl, usefbcon, costfct,
                     nochannels, patnorm, usetvref, tv_alpha, tv_gamma, tv_delta, tv_innerit, tv_solverit, tv_sor,
                     verbosity, nop);
  } catch (const std::exception& e) {
    fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  if (verbosity > 1) gettimeofday(&tv, NULL);

  // *** resize to original scale, crop, save (run_dense.cpp:406-421)
  if (lv_l != 0) {
    for (float& v : flowout.px) v = v * (float)sc_fct;
    flowout = upsample_linear(flowout, sc_fct);
  }
  ImageF out;
  out.w = width_org;
  out.h = height_org;
  out.c = nop;
  out.px.resize((size_t)out.w * out.h * nop);
  const int ox = (int)floor((float)padw / 2.0f), oy = (int)floor((float)padh / 2.0f);
  for (int y = 0; y < out.h; ++y)
    for (int x = 0; x < out.w; ++x)
      for (int k = 0; k < nop; ++k) out.at(x, y, k) = flowout.at(x + ox, y + oy, k);
  if (SELECTMODE == 1) SaveFlowFile(out, outfile);
  else SavePFMFile(out, outfile);
  if (verbosity > 1) printf("TIME (Saving flow file  ) (ms): %3g\n", elapsed_ms(tv));
  return 0;
}
#endif  // OFDIS_BATCH
