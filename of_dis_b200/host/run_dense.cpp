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
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
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
  int maxb = 64, first_num = 2;
  bool warm = false, batch_set = false, bidir = false, kitti = false, color = false;
  float color_max = 0.0f;  // --color-max; 0: every pair's own maximum
  const char* color_max_arg = nullptr;
  const char* interp_arg = nullptr;  // --interpolate T
  float interp_t = 0.0f;
  const char* gtlist = nullptr;
  const char* tracks_path = nullptr;  // --tracks PATH
  const char* desc_path = nullptr;    // --descriptors PATH
  const char* fisher_arg[2] = {nullptr, nullptr};  // --fisher CODEBOOK PATH
  bool lr_check = false, disp_fill = false;  // --lr-check, --fill
  const char* speckle_arg[2] = {nullptr, nullptr};  // --speckle N R
  const char* camera_arg = nullptr;  // --camera fx,fy,cx,cy,baseline,doffs
  const char* gm_arg[2] = {nullptr, nullptr};  // --global-motion MODEL PATH
  const char* stab_arg[3] = {nullptr, nullptr, nullptr};  // --stabilize RADIUS CROP DIR
  const char* sf_list = nullptr;    // --scene-flow DISPLIST
  const char* sf_gtlist = nullptr;  // --gt-scene-flow GTLIST
  const char* odo_dir = nullptr;     // --odometry DIR
  const char* odo_gtlist = nullptr;  // --gt-poses LIST
  const char* fuse_arg = nullptr;    // --fuse voxel,trunc,x0,y0,z0,nx,ny,nz
  bool fuse_mesh = false;            // --mesh
  for (;;) {
    if (argc >= first_num + 2 && !strcmp(argv[first_num], "--batch")) {
      maxb = atoi(argv[first_num + 1]);
      first_num += 2;
      batch_set = true;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--warm-start")) {
      warm = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--bidirectional")) {
      bidir = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--kitti")) {
      kitti = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--color")) {
      color = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--color-max")) {
      if (argc < first_num + 2 || color_max_arg) {
        fprintf(stderr, "error: --color-max takes one positive number\n");
        return 2;
      }
      color_max_arg = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--interpolate")) {
      if (argc < first_num + 2 || interp_arg) {
        fprintf(stderr, "error: --interpolate takes one time between 0 and 1\n");
        return 2;
      }
      interp_arg = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--tracks")) {
      if (argc < first_num + 2 || tracks_path) {
        fprintf(stderr, "error: --tracks takes one output path\n");
        return 2;
      }
      tracks_path = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--descriptors")) {
      if (argc < first_num + 2 || desc_path) {
        fprintf(stderr, "error: --descriptors takes one output path\n");
        return 2;
      }
      desc_path = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--fisher")) {
      if (argc < first_num + 3 || fisher_arg[0]) {
        fprintf(stderr, "error: --fisher takes a codebook file and an output path\n");
        return 2;
      }
      fisher_arg[0] = argv[first_num + 1];
      fisher_arg[1] = argv[first_num + 2];
      first_num += 3;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--lr-check")) {
      lr_check = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--fill")) {
      disp_fill = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--speckle")) {
      if (argc < first_num + 3 || speckle_arg[0]) {
        fprintf(stderr, "error: --speckle takes a size N and a difference R\n");
        return 2;
      }
      speckle_arg[0] = argv[first_num + 1];
      speckle_arg[1] = argv[first_num + 2];
      first_num += 3;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--camera")) {
      if (argc < first_num + 2 || camera_arg) {
        fprintf(stderr, "error: --camera takes fx,fy,cx,cy,baseline,doffs\n");
        return 2;
      }
      camera_arg = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--global-motion")) {
      if (argc < first_num + 3 || gm_arg[0]) {
        fprintf(stderr, "error: --global-motion takes a model (similarity, affine or homography) and an output path\n");
        return 2;
      }
      gm_arg[0] = argv[first_num + 1];
      gm_arg[1] = argv[first_num + 2];
      first_num += 3;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--stabilize")) {
      if (argc < first_num + 4 || stab_arg[0]) {
        fprintf(stderr, "error: --stabilize takes a radius, a crop and an output directory\n");
        return 2;
      }
      stab_arg[0] = argv[first_num + 1];
      stab_arg[1] = argv[first_num + 2];
      stab_arg[2] = argv[first_num + 3];
      first_num += 4;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--scene-flow")) {
      if (argc < first_num + 2 || sf_list) {
        fprintf(stderr, "error: --scene-flow takes one disparity list file\n");
        return 2;
      }
      sf_list = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--gt-scene-flow")) {
      if (argc < first_num + 2 || sf_gtlist) {
        fprintf(stderr, "error: --gt-scene-flow takes one ground-truth list file\n");
        return 2;
      }
      sf_gtlist = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--odometry")) {
      if (argc < first_num + 2 || odo_dir) {
        fprintf(stderr, "error: --odometry takes one output directory\n");
        return 2;
      }
      odo_dir = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--fuse")) {
      if (argc < first_num + 2 || fuse_arg) {
        fprintf(stderr, "error: --fuse takes voxel,trunc,x0,y0,z0,nx,ny,nz\n");
        return 2;
      }
      fuse_arg = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--mesh")) {
      fuse_mesh = true;
      first_num += 1;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--gt-poses")) {
      if (argc < first_num + 2 || odo_gtlist) {
        fprintf(stderr, "error: --gt-poses takes one list of KITTI poses files\n");
        return 2;
      }
      odo_gtlist = argv[first_num + 1];
      first_num += 2;
    } else if (argc >= first_num + 1 && !strcmp(argv[first_num], "--gt")) {
      if (argc < first_num + 2 || gtlist) {
        fprintf(stderr, "error: --gt takes one ground-truth list file\n");
        return 2;
      }
      gtlist = argv[first_num + 1];
      first_num += 2;
    } else {
      break;
    }
  }
  if (warm && batch_set) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --batch\n");
    return 2;
  }
  if (warm && bidir) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --bidirectional\n");
    return 2;
  }
  if (warm && interp_arg) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --interpolate\n");
    return 2;
  }
  if (warm && tracks_path) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --tracks\n");
    return 2;
  }
  if (sf_list && SELECTMODE != 1) {
    fprintf(stderr, "error: --scene-flow joins flows with disparities; the stereo binaries take no --scene-flow\n");
    return 2;
  }
  if (sf_list && warm) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --scene-flow\n");
    return 2;
  }
  if (sf_gtlist && !sf_list) {
    fprintf(stderr, "error: --gt-scene-flow evaluates the scene flow of --scene-flow; give --scene-flow too\n");
    return 2;
  }
  if (odo_dir && SELECTMODE != 1) {
    fprintf(stderr, "error: --odometry fits the rig's motion from flows; the stereo binaries take no --odometry\n");
    return 2;
  }
  if (odo_dir && warm) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --odometry\n");
    return 2;
  }
  if (odo_dir && (!sf_list || !camera_arg)) {
    fprintf(stderr, "error: --odometry needs the disparities of --scene-flow and the stereo camera of --camera\n");
    return 2;
  }
  if (odo_gtlist && !odo_dir) {
    fprintf(stderr, "error: --gt-poses evaluates the poses of --odometry; give --odometry too\n");
    return 2;
  }
  if (fuse_arg && SELECTMODE != 1) {
    fprintf(stderr, "error: --fuse places disparities with the poses of --odometry; the stereo binaries take no --fuse\n");
    return 2;
  }
  if (fuse_arg && warm) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --fuse\n");
    return 2;
  }
  if (fuse_arg && !odo_dir) {
    fprintf(stderr, "error: --fuse places disparities with the poses of --odometry; give --odometry too\n");
    return 2;
  }
  if (fuse_mesh && !fuse_arg) {
    fprintf(stderr, "error: --mesh meshes the volume of --fuse; give --fuse too\n");
    return 2;
  }
  ofdis_fuse_params fuse_p;
  memset(&fuse_p, 0, sizeof(fuse_p));
  if (fuse_arg) {
    double v[8];
    const char* q = fuse_arg;
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
    if (!ok) {
      fprintf(stderr, "error: --fuse takes eight numbers voxel,trunc,x0,y0,z0,nx,ny,nz with voxel and trunc > 0, "
                      "integer sizes >= 1 and at most 2^30 voxels, got %s\n", fuse_arg);
      return 2;
    }
    fuse_p.voxel = (float)v[0];
    fuse_p.trunc = (float)v[1];
    for (int e = 0; e < 3; ++e) fuse_p.origin[e] = (float)v[2 + e];
    fuse_p.nx = (int)v[5];
    fuse_p.ny = (int)v[6];
    fuse_p.nz = (int)v[7];
    fuse_p.max_weight = 64.0f;
    fuse_p.color = 1;
  }
  // --camera on a flow binary belongs to --scene-flow
  const bool disp_on = lr_check || disp_fill || speckle_arg[0] || (camera_arg && !sf_list);
  if (disp_on && SELECTMODE == 1) {
    fprintf(stderr, "error: --lr-check, --speckle, --fill and --camera filter stereo disparities; the flow binaries "
                    "take none of them\n");
    return 2;
  }
  if (warm && disp_on) {
    fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --lr-check, --speckle, --fill or --camera\n");
    return 2;
  }
  int gm_model = 0;  // --global-motion: OFDIS_MOTION_*
  if (gm_arg[0]) {
    if (SELECTMODE != 1) {
      fprintf(stderr, "error: --global-motion fits the camera motion of flows; the stereo binaries take no "
                      "--global-motion\n");
      return 2;
    }
    if (warm) {
      fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --global-motion\n");
      return 2;
    }
    gm_model = !strcmp(gm_arg[0], "similarity") ? OFDIS_MOTION_SIMILARITY
               : !strcmp(gm_arg[0], "affine")   ? OFDIS_MOTION_AFFINE
               : !strcmp(gm_arg[0], "homography") ? OFDIS_MOTION_HOMOGRAPHY : 0;
    if (!gm_model) {
      fprintf(stderr, "error: --global-motion takes the model similarity, affine or homography, got %s\n", gm_arg[0]);
      return 2;
    }
  }
  if (desc_path) {
    if (SELECTMODE != 1) {
      fprintf(stderr, "error: --descriptors describes the tracks of flows; the stereo binaries take no --descriptors\n");
      return 2;
    }
    if (warm) {
      fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --descriptors\n");
      return 2;
    }
    if (!tracks_path) {
      fprintf(stderr, "error: --descriptors describes the clips of --tracks; give --tracks too\n");
      return 2;
    }
  }
  if (fisher_arg[0]) {
    if (SELECTMODE != 1) {
      fprintf(stderr, "error: --fisher encodes the descriptors of flows; the stereo binaries take no --fisher\n");
      return 2;
    }
    if (warm) {
      fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --fisher\n");
      return 2;
    }
    if (!tracks_path) {
      fprintf(stderr, "error: --fisher encodes the clips of --tracks; give --tracks too\n");
      return 2;
    }
  }
  ofdis_traj_params trp;  // --descriptors, --fisher: Wang and Schmid's settings
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
  const int tdim = 2 * trp.L + trp.ns * trp.ns * trp.nt * 33;
  FisherBook fbook;  // --fisher: the codebook, whose blocks must be the descriptors' (shape, HOG, HOF, MBHx, MBHy)
  if (fisher_arg[0]) {
    string err;
    if (!read_fisher_book(fisher_arg[0], fbook, err)) {
      fprintf(stderr, "error: %s: %s\n", fisher_arg[0], err.c_str());
      return 2;
    }
    const int c = trp.nt * trp.ns * trp.ns, din[5] = {2 * trp.L, 8 * c, 9 * c, 8 * c, 8 * c};
    bool match = fbook.cb.desc_dim == tdim && fbook.cb.nblocks == 5;
    for (int b = 0, off = 0; match && b < 5; off += din[b++])
      match = fbook.cb.blocks[b].offset == off && fbook.cb.blocks[b].dim_in == din[b];
    if (!match) {
      fprintf(stderr, "error: %s: the codebook's blocks are not the descriptors' (desc_dim %d, blocks 0+%d, %d+%d, "
                      "%d+%d, %d+%d, %d+%d)\n", fisher_arg[0], tdim, din[0], din[0], din[1], din[0] + din[1], din[2],
              din[0] + din[1] + din[2], din[3], tdim - din[4], din[4]);
      return 2;
    }
  }
  const bool traj_stage = desc_path || fisher_arg[0];  // the descriptor stage runs in place of the tracker's calls
  ofdis_stab_params stp;  // --stabilize
  memset(&stp, 0, sizeof(stp));
  vector<double> stab_wts;
  if (stab_arg[0]) {
    if (SELECTMODE != 1) {
      fprintf(stderr, "error: --stabilize smooths the camera motion of flows; the stereo binaries take no --stabilize\n");
      return 2;
    }
    if (warm) {
      fprintf(stderr, "error: --warm-start runs one pair per launch; it takes no --stabilize\n");
      return 2;
    }
    if (!gm_arg[0]) {
      fprintf(stderr, "error: --stabilize smooths the models of --global-motion; give --global-motion too\n");
      return 2;
    }
    char *e0 = nullptr, *e1 = nullptr;
    const long r = strtol(stab_arg[0], &e0, 10);
    const float crop = strtof(stab_arg[1], &e1);
    if (e0 == stab_arg[0] || *e0 || r < 1 || r > 64 || e1 == stab_arg[1] || *e1 || !(crop >= 0.0f && crop < 0.5f)) {
      fprintf(stderr, "error: --stabilize takes a radius 1..64 and a crop 0 <= CROP < 0.5, got %s %s\n", stab_arg[0],
              stab_arg[1]);
      return 2;
    }
    stp.radius = (int)r;
    stp.crop = crop;
    stp.limit = crop > 0.0f ? 1 : 0;
    for (int d = 0; d <= stp.radius; ++d) stab_wts.push_back(exp(-(double)(d * d) / (2.0 * stp.radius)));
  }
  ofdis_disp_filter dfilt;
  memset(&dfilt, 0, sizeof(dfilt));
  dfilt.lr_check = lr_check ? 1 : 0;
  dfilt.alpha = 0.0f;
  dfilt.beta = 1.0f;
  dfilt.speckle_diff = 1.0f;
  dfilt.fill = disp_fill ? 1 : 0;
  if (speckle_arg[0]) {
    char *e0 = nullptr, *e1 = nullptr;
    const long sz = strtol(speckle_arg[0], &e0, 10);
    const float diff = strtof(speckle_arg[1], &e1);
    if (e0 == speckle_arg[0] || *e0 || sz < 1 || sz > INT_MAX || e1 == speckle_arg[1] || *e1 ||
        !(diff >= 0.0f && diff <= FLT_MAX)) {
      fprintf(stderr, "error: --speckle takes a size N >= 1 and a finite difference R >= 0, got %s %s\n", speckle_arg[0],
              speckle_arg[1]);
      return 2;
    }
    dfilt.speckle_size = (int)sz;
    dfilt.speckle_diff = diff;
  }
  ofdis_stereo_camera dcam;
  memset(&dcam, 0, sizeof(dcam));
  if (camera_arg) {
    float v[6];
    const char* q = camera_arg;
    bool ok = true;
    for (int i = 0; i < 6 && ok; ++i) {
      char* end = nullptr;
      v[i] = strtof(q, &end);
      ok = end != q && (i < 5 ? *end == ',' : *end == 0) && v[i] >= -FLT_MAX && v[i] <= FLT_MAX;
      q = end + (i < 5 ? 1 : 0);
    }
    if (!ok || !(v[0] > 0.0f) || !(v[1] > 0.0f) || !(v[4] > 0.0f)) {
      fprintf(stderr, "error: --camera takes six finite numbers fx,fy,cx,cy,baseline,doffs with fx, fy and baseline "
                      "> 0, got %s\n", camera_arg);
      return 2;
    }
    dcam = ofdis_stereo_camera{v[0], v[1], v[2], v[3], v[4], v[5]};
  }
  if (interp_arg) {
    char* end = nullptr;
    interp_t = strtof(interp_arg, &end);
    if (end == interp_arg || *end || !(interp_t > 0.0f && interp_t < 1.0f)) {
      fprintf(stderr, "error: --interpolate takes a time T with 0 < T < 1, got %s\n", interp_arg);
      return 2;
    }
  }
  // --interpolate and --tracks need the backward flows: the backward slots run whenever one of them is given
  const bool two_way = bidir || interp_arg || tracks_path || lr_check;
  if (color_max_arg) {
    char* end = nullptr;
    color_max = strtof(color_max_arg, &end);
    if (!color) {
      fprintf(stderr, "error: --color-max needs --color\n");
      return 2;
    }
    if (end == color_max_arg || *end || !(color_max > 0.0f && color_max <= FLT_MAX)) {
      fprintf(stderr, "error: --color-max takes a positive finite number, got %s\n", color_max_arg);
      return 2;
    }
  }
  if (warm) maxb = 1;
  const int nnum = argc - first_num;
  if (maxb < 1 || (nnum > 1 && nnum != 20)) {
    fprintf(stderr, "error: expected 0, 1 or exactly 20 numbers, got %d\n", nnum);
    return 2;
  }
  struct Job { string a, b, out; };
  vector<Job> jobs;
  {
    FILE* f = fopen(argv[1], "r");
    if (!f) {
      fprintf(stderr, "error: cannot read %s\n", argv[1]);
      return 1;
    }
    char a[4096], b[4096], o[4096];
    while (fscanf(f, "%4095s %4095s %4095s", a, b, o) == 3) jobs.push_back({a, b, o});
    fclose(f);
  }
  const int nochannels = (SELECTCHANNEL == 3) ? 3 : 1;
  const int nop = (SELECTMODE == 1) ? 2 : 1;
  // --gt: the list, then every file against its pair's image size, before any device work
  vector<string> gts;
  if (gtlist) {
    FILE* f = fopen(gtlist, "r");
    if (!f) {
      fprintf(stderr, "error: cannot read %s\n", gtlist);
      return 1;
    }
    char g[4096];
    while (fscanf(f, "%4095s", g) == 1) gts.push_back(g);
    fclose(f);
    if (gts.size() != jobs.size()) {
      fprintf(stderr, "error: --gt: %s lists %zu ground-truth files for %zu pairs\n", gtlist, gts.size(), jobs.size());
      return 2;
    }
    vector<float> gtf;
    for (size_t k = 0; k < jobs.size(); ++k) {
      int iw = 0, ih = 0;
      string err;
      if (!image_size(jobs[k].a.c_str(), iw, ih)) {
        fprintf(stderr, "error: cannot read the pair %s %s (binary PGM/PPM or 8-bit PNG of equal size)\n",
                jobs[k].a.c_str(), jobs[k].b.c_str());
        return 1;
      }
      if (!read_gt_file(gts[k].c_str(), iw, ih, nop, gtf, err)) {
        fprintf(stderr, "error: %s: %s\n", gts[k].c_str(), err.c_str());
        return 1;
      }
    }
  }
  // --scene-flow / --gt-scene-flow: two and three files per pair, each checked against its pair's image size before
  // any device work
  vector<string> sf_files, sf_gts;
  for (int li = 0; li < 2; ++li) {
    const char* list = li ? sf_gtlist : sf_list;
    vector<string>& files = li ? sf_gts : sf_files;
    const size_t per = li ? 3 : 2;
    if (!list) continue;
    FILE* f = fopen(list, "r");
    if (!f) {
      fprintf(stderr, "error: cannot read %s\n", list);
      return 1;
    }
    char g[4096];
    while (fscanf(f, "%4095s", g) == 1) files.push_back(g);
    fclose(f);
    if (files.size() != per * jobs.size()) {
      fprintf(stderr, "error: %s: %s lists %zu files for %zu pairs (%zu per pair)\n",
              li ? "--gt-scene-flow" : "--scene-flow", list, files.size(), jobs.size(), per);
      return 2;
    }
    vector<float> tmp;
    for (size_t k = 0; k < files.size(); ++k) {
      int iw = 0, ih = 0;
      string err;
      const Job& jb = jobs[k / per];
      if (!image_size(jb.a.c_str(), iw, ih)) {
        fprintf(stderr, "error: cannot read the pair %s %s (binary PGM/PPM or 8-bit PNG of equal size)\n", jb.a.c_str(),
                jb.b.c_str());
        return 1;
      }
      if (!read_gt_file(files[k].c_str(), iw, ih, li && k % 3 == 2 ? 2 : 1, tmp, err)) {
        fprintf(stderr, "error: %s: %s\n", files[k].c_str(), err.c_str());
        return 2;
      }
    }
  }
  // --odometry: the clip and frame of every pair, the ground-truth poses of every clip and the output files, before
  // any device work
  vector<int> odo_clip(jobs.size(), 0), odo_frame(jobs.size(), 0);
  vector<vector<double>> odo_gt;  // per clip, 12 numbers per line
  vector<vector<double>> odo_rel;  // per clip, 12 numbers per pair (filled as the pairs are computed)
  FILE* odo_file = nullptr;
  if (odo_dir) {
    int nclips = 0;
    for (size_t k = 0; k < jobs.size(); ++k) {
      const bool cont = k > 0 && jobs[k].a == jobs[k - 1].b;
      odo_clip[k] = cont ? odo_clip[k - 1] : nclips++;
      odo_frame[k] = cont ? odo_frame[k - 1] + 1 : 0;
    }
    odo_rel.resize(nclips);
    if (odo_gtlist) {
      FILE* f = fopen(odo_gtlist, "r");
      if (!f) {
        fprintf(stderr, "error: cannot read %s\n", odo_gtlist);
        return 2;
      }
      vector<string> files;
      char g[4096];
      while (fscanf(f, "%4095s", g) == 1) files.push_back(g);
      fclose(f);
      if ((int)files.size() != nclips) {
        fprintf(stderr, "error: --gt-poses: %s lists %zu poses files for %d clips\n", odo_gtlist, files.size(), nclips);
        return 2;
      }
      vector<int> need(nclips, 0);
      for (size_t k = 0; k < jobs.size(); ++k) need[odo_clip[k]] = odo_frame[k] + 2;
      for (int c = 0; c < nclips; ++c) {
        FILE* pf = fopen(files[c].c_str(), "r");
        if (!pf) {
          fprintf(stderr, "error: cannot read %s\n", files[c].c_str());
          return 2;
        }
        vector<double> v;
        double x;
        while (fscanf(pf, "%lf", &x) == 1) v.push_back(x);
        const bool eof = feof(pf);
        fclose(pf);
        if (!eof || v.size() % 12 || (int)(v.size() / 12) < need[c]) {
          fprintf(stderr, "error: %s: a KITTI poses file of at least %d lines of 12 numbers, got %zu numbers\n",
                  files[c].c_str(), need[c], v.size());
          return 2;
        }
        odo_gt.push_back(v);
      }
    }
    const string path = string(odo_dir) + "/odometry.txt";
    odo_file = fopen(path.c_str(), "w");
    if (!odo_file) {
      fprintf(stderr, "error: --odometry: cannot write %s\n", path.c_str());
      return 2;
    }
  }
  double odo_terr = 0.0, odo_rerr = 0.0;
  size_t odo_eval = 0;
  vector<double> odo_pose;
  vector<ofdis_motion_stats> odo_stats;
  vector<uint8_t> odo_mask;
  vector<float> odo_om;
  double fuse_T[12];              // --fuse: the chained pose of the clip's next image1
  int fuse_frames = 0;            // frames pushed into the clip's volume
  vector<double> fuse_poses;
  vector<ofdis_fuse_point> fuse_pts;
  vector<unsigned int> fuse_faces;  // --mesh
  // --descriptors, --fisher: every pair's frames hold an N x N patch, checked before any device work
  for (size_t k = 0; k < jobs.size() && traj_stage; ++k) {
    int iw = 0, ih = 0;
    if (!image_size(jobs[k].a.c_str(), iw, ih)) {
      fprintf(stderr, "error: cannot read the pair %s %s (binary PGM/PPM or 8-bit PNG of equal size)\n",
              jobs[k].a.c_str(), jobs[k].b.c_str());
      return 1;
    }
    if (iw < trp.N || ih < trp.N) {
      fprintf(stderr, "error: --%s needs frames of at least %d x %d, %s is %d x %d\n",
              desc_path ? "descriptors" : "fisher", trp.N, trp.N, jobs[k].a.c_str(), iw, ih);
      return 2;
    }
  }
  FILE* desc_file = nullptr;
  if (desc_path) {
    desc_file = fopen(desc_path, "w");
    if (!desc_file) {
      fprintf(stderr, "error: cannot write %s\n", desc_path);
      return 1;
    }
    fprintf(desc_file, "# clip id start mean_x mean_y sd_x sd_y length d0 .. d%d\n", tdim - 1);
  }
  FILE* fisher_file = nullptr;
  int fv_floats = 0;
  if (fisher_arg[0]) {
    fisher_file = fopen(fisher_arg[1], "w");
    if (!fisher_file) {
      fprintf(stderr, "error: cannot write %s\n", fisher_arg[1]);
      if (desc_file) fclose(desc_file);
      return 1;
    }
    for (int b = 0; b < fbook.cb.nblocks; ++b) fv_floats += 2 * fbook.cb.K * fbook.cb.blocks[b].dim;
    fprintf(fisher_file, "# clip n_desc n_0 .. n_%d fv0 .. fv%d\n", fbook.cb.nblocks - 1, fv_floats - 1);
  }
  FILE* tracks_file = nullptr;
  if (tracks_path) {
    tracks_file = fopen(tracks_path, "w");
    if (!tracks_file) {
      fprintf(stderr, "error: cannot write %s\n", tracks_path);
      if (desc_file) fclose(desc_file);
      if (fisher_file) fclose(fisher_file);
      return 1;
    }
    fprintf(tracks_file, "# clip frame id x y\n");
  }
  FILE* stab_file = nullptr;
  const string stab_txt = stab_arg[0] ? string(stab_arg[2]) + "/stab.txt" : string();
  if (stab_arg[0]) {
    stab_file = fopen(stab_txt.c_str(), "w");
    if (!stab_file) {
      fprintf(stderr, "error: cannot write %s\n", stab_txt.c_str());
      if (tracks_file) fclose(tracks_file);
      if (desc_file) fclose(desc_file);
      if (fisher_file) fclose(fisher_file);
      return 1;
    }
  }
  FILE* gm_file = nullptr;
  if (gm_model) {
    gm_file = fopen(gm_arg[1], "w");
    if (!gm_file) {
      fprintf(stderr, "error: cannot write %s\n", gm_arg[1]);
      if (tracks_file) fclose(tracks_file);
      if (desc_file) fclose(desc_file);
      if (fisher_file) fclose(fisher_file);
      if (stab_file) fclose(stab_file);
      return 1;
    }
  }
  const int nclasses = bidir ? 3 : 1;  // with --bidirectional the forward consistency mask's classes
  vector<ofdis_error_stats> eval_total(nclasses + 1), eval_pairs;  // [0]: all pixels, [1 + c]: class c
  memset(eval_total.data(), 0, sizeof(ofdis_error_stats) * eval_total.size());
  vector<float> gt_batch, gt_one;
  // --scene-flow: the batch's disparities, ground truth and outputs; the totals ([0]: all pixels, [1 + c]: class c)
  vector<float> sf_d0, sf_d1, sf_g0, sf_g1, sf_gf, sf_w, sf_m;
  vector<ofdis_sf_stats> sf_pairs, sf_total(nclasses + 1);
  memset(sf_total.data(), 0, sizeof(ofdis_sf_stats) * sf_total.size());
  timeval tv;
  gettimeofday(&tv, NULL);
  size_t done = 0, seq_pairs = 0, seq_decoded = 0, warm_pairs = 0;
  ofdis_ctx* ctx = nullptr;
  int ctx_w = -1, ctx_h = -1, verbosity = 0;
  vector<uint8_t> frames;
  vector<float> flows;
  vector<uint16_t> kflows;  // --kitti: the encoded slots
  vector<uint8_t> masks;
  vector<uint8_t> colors;  // --color: the color images of the slots
  vector<uint8_t> interp, interp_png;  // --interpolate: the frames at time T, one written as RGB
  vector<float> ddisp, ddepth, dxyz;  // --lr-check / --speckle / --fill / --camera: the filtered outputs
  vector<uint8_t> dstatus, dply;
  vector<double> gm_models;  // --global-motion: the models, stats and per-pixel outputs of the batch
  vector<ofdis_motion_stats> gm_stats;
  vector<uint8_t> gm_mask, gm_reg, gm_png;
  vector<float> gm_res;
  Image8 last;  // image2 of the previous batch's last pair
  // --tracks: the tracker's points and counts, the clip being tracked (-1 none) and its next frame, the totals of the
  // finished clips
  vector<ofdis_track_point> tpoints;
  vector<int> tcounts;
  int tclip = -1, tframe = 0;
  size_t tframes = 0;
  ofdis_track_stats ttotal;
  memset(&ttotal, 0, sizeof(ttotal));
  // --descriptors: the segments of a call and the totals of the finished clips
  vector<ofdis_traj_record> trec;
  vector<float> tdesc;
  vector<int> tndesc;
  ofdis_traj_stats dtotal;
  memset(&dtotal, 0, sizeof(dtotal));
  // --fisher: whether the clip's encoder is live, the vector of a take, the totals, the status of the last take
  bool fisher_live = false;
  vector<float> fvec(fv_floats);
  long long fpushed = 0, fskipped[OFDIS_FISHER_MAX_BLOCKS] = {0};
  int fclips = 0, fisher_rc = OFDIS_OK;
  auto end_clip = [&]() {  // adds the tracked clip's counters to the totals; --fisher: takes the clip's vector
    if (fisher_live) {
      fisher_live = false;
      ofdis_fisher_stats fs;
      fisher_rc = ofdis_fisher_take(ctx, fvec.data(), nullptr, &fs, OFDIS_MEM_HOST);
      if (fisher_rc == OFDIS_OK) {
        fprintf(fisher_file, "%d %lld", tclip, fs.pushed);
        for (int b = 0; b < fbook.cb.nblocks; ++b) fprintf(fisher_file, " %lld", fs.n[b]);
        for (int i = 0; i < fv_floats; ++i) fprintf(fisher_file, " %.9g", (double)fvec[i]);
        fprintf(fisher_file, "\n");
        ++fclips;
        fpushed += fs.pushed;
        for (int b = 0; b < fbook.cb.nblocks; ++b) fskipped[b] += fs.skipped[b];
      }
    }
    ofdis_track_stats st;
    if (tclip < 0 || ofdis_track_stats_get(ctx, &st) != OFDIS_OK) return;
    ttotal.seeded += st.seeded;
    ttotal.ended_leaves += st.ended_leaves;
    ttotal.ended_inconsistent += st.ended_inconsistent;
    ttotal.ended_boundary += st.ended_boundary;
    ttotal.dropped += st.dropped;
    ofdis_traj_stats ds;
    if (!traj_stage || ofdis_traj_stats_get(ctx, &ds) != OFDIS_OK) return;
    dtotal.emitted += ds.emitted;
    dtotal.rejected_static += ds.rejected_static;
    dtotal.rejected_erratic += ds.rejected_erratic;
    dtotal.rejected_jump += ds.rejected_jump;
    dtotal.rejected_camera += ds.rejected_camera;
  };
  auto write_desc = [&](int count) {
    for (int i = 0; i < count; ++i) {
      const ofdis_traj_record& r = trec[i];
      fprintf(desc_file, "%d %d %d %.9g %.9g %.9g %.9g %.9g", tclip, r.id, r.start, (double)r.mean_x, (double)r.mean_y,
              (double)r.sd_x, (double)r.sd_y, (double)r.length);
      const float* d = tdesc.data() + (size_t)i * tdim;
      for (int e = 0; e < tdim; ++e) fprintf(desc_file, " %.9g", (double)d[e]);
      fprintf(desc_file, "\n");
    }
  };
  // --stabilize: the emitted frames and records, the clip being stabilised (-1 none), whether its stabiliser is live
  // and its frame size
  vector<uint8_t> sbuf, spng;
  vector<ofdis_stab_frame> sinfo;
  int sclip = -1, sw = 0, sh = 0;
  bool stab_live = false;
  auto write_stab = [&](int count) {
    const size_t shwc = (size_t)sw * sh * nochannels;
    for (int i = 0; i < count; ++i) {
      const ofdis_stab_frame& f = sinfo[i];
      fprintf(stab_file, "%d %lld", sclip, f.frame);
      for (int e = 0; e < 9; ++e) fprintf(stab_file, " %.17g", f.correction[e]);
      fprintf(stab_file, " %.17g %d\n", f.lambda, f.status);
      const uint8_t* im = sbuf.data() + (size_t)i * shwc;
      if (nochannels == 3) {  // the decoder's BGR -> RGB
        spng.resize(shwc);
        for (size_t q = 0; q < shwc; q += 3) {
          spng[q] = im[q + 2];
          spng[q + 1] = im[q + 1];
          spng[q + 2] = im[q];
        }
        im = spng.data();
      }
      char name[64];
      snprintf(name, sizeof(name), "/stab_%04d_%06lld.png", sclip, f.frame);
      save_png(im, sw, sh, nochannels, 8, (string(stab_arg[2]) + name).c_str());
    }
  };
  auto stab_end = [&]() -> int {  // emits the rest of the clip being stabilised
    if (!stab_live) return OFDIS_OK;
    stab_live = false;
    sbuf.resize((size_t)stp.radius * sw * sh * nochannels);
    sinfo.resize(stp.radius);
    int count = 0;
    const int rc = ofdis_stab_finish(ctx, sbuf.data(), sinfo.data(), &count, OFDIS_MEM_HOST);
    if (rc == OFDIS_OK) write_stab(count);
    return rc;
  };
  auto write_tracks = [&](const ofdis_track_point* p, int count) {
    for (int i = 0; i < count; ++i)
      fprintf(tracks_file, "%d %d %d %.9g %.9g\n", tclip, tframe, p[i].id, (double)p[i].x, (double)p[i].y);
    ++tframe;
    ++tframes;
  };
  size_t j0 = 0;
  while (j0 < jobs.size()) {
    // load up to maxb pairs of one size; a frame that continues the previous pair is not decoded again
    vector<Image8> imgs;  // decoded frames of this batch
    vector<int> ia, ib;   // per pair: indices of image1, image2 in imgs
    int w = 0, h = 0, n = 0, decoded = 0;
    while (j0 + n < jobs.size() && n < maxb) {
      const Job& jb = jobs[j0 + n];
      const bool in_batch = n > 0 && jb.a == jobs[j0 + n - 1].b;          // image1 = this batch's last frame
      const bool from_last = n == 0 && j0 > 0 && jb.a == jobs[j0 - 1].b;  // image1 = the previous batch's last frame
      Image8 a8, b8;
      if (from_last) a8 = last;
      const bool ok = in_batch || from_last || load_image(jb.a.c_str(), nochannels, a8);
      const Image8& ra = in_batch ? imgs[ib.back()] : a8;
      if (!ok || !load_image(jb.b.c_str(), nochannels, b8) || ra.w != b8.w || ra.h != b8.h) {
        fprintf(stderr, "error: cannot read the pair %s %s (binary PGM/PPM or 8-bit PNG of equal size)\n",
                jb.a.c_str(), jb.b.c_str());
        if (ctx) ofdis_destroy(ctx);
        return 1;
      }
      if (n == 0) { w = b8.w; h = b8.h; }
      else if (b8.w != w || b8.h != h) break;  // next group
      if (in_batch) ia.push_back(ib.back());
      else {
        decoded += from_last ? 0 : 1;
        ia.push_back((int)imgs.size());
        imgs.push_back(std::move(a8));
      }
      ib.push_back((int)imgs.size());
      imgs.push_back(std::move(b8));
      ++decoded;
      ++n;
    }
    bool seq = n >= 2;
    for (int k = 1; k < n && seq; ++k) seq = ia[k] == ib[k - 1];
    frames.clear();
    if (seq) {
      frames.insert(frames.end(), imgs[ia[0]].px.begin(), imgs[ia[0]].px.end());
      for (int k = 0; k < n; ++k) frames.insert(frames.end(), imgs[ib[k]].px.begin(), imgs[ib[k]].px.end());
      seq_pairs += n;
      seq_decoded += decoded;
    } else {
      for (int k = 0; k < n; ++k) {
        frames.insert(frames.end(), imgs[ia[k]].px.begin(), imgs[ia[k]].px.end());
        frames.insert(frames.end(), imgs[ib[k]].px.begin(), imgs[ib[k]].px.end());
      }
      for (int k = 0; k < n && two_way; ++k) {  // the swapped copies
        frames.insert(frames.end(), imgs[ib[k]].px.begin(), imgs[ib[k]].px.end());
        frames.insert(frames.end(), imgs[ia[k]].px.begin(), imgs[ia[k]].px.end());
      }
    }
    last = std::move(imgs[ib.back()]);
    CliParams P;
    parse_cli_params(nnum, argv + first_num, w, P);
    verbosity = P.verbosity;
    if (w != ctx_w || h != ctx_h) {
      end_clip();  // a pair of another size never continues the previous one
      if (fisher_rc != OFDIS_OK || stab_end() != OFDIS_OK) {
        fprintf(stderr, "error: %s\n", ofdis_last_error(ctx));
        ofdis_destroy(ctx);
        return 1;
      }
      if (ctx) ofdis_destroy(ctx);
      ctx = nullptr;
      ofdis_params p;
      memset(&p, 0, sizeof(p));
      p.sc_f = P.lv_f; p.sc_l = P.lv_l; p.max_iter = P.maxiter; p.min_iter = P.miniter;
      p.dp_thresh = P.mindprate; p.dr_thresh = P.mindrrate; p.res_thresh = P.minimgerr;
      p.p_samp_s = P.patchsz; p.patove = P.poverl; p.usefbcon = P.usefbcon ? 1 : 0; p.costfct = P.costfct;
      p.noc = nochannels; p.patnorm = P.patnorm; p.usetvref = P.usetvref ? 1 : 0;
      p.tv_alpha = P.tv_alpha; p.tv_gamma = P.tv_gamma; p.tv_delta = P.tv_delta;
      p.tv_innerit = P.tv_innerit; p.tv_solverit = P.tv_solverit; p.tv_sor = P.tv_sor; p.verbosity = P.verbosity;
      const int scf = 1 << (warm ? P.lv_f + 1 : P.lv_f);
      const int rc = ofdis_create(&ctx, 0, nullptr, &p, nop, (w + scf - 1) / scf * scf, (h + scf - 1) / scf * scf,
                                  P.patchsz, two_way ? 2 * maxb : maxb);
      if (rc != OFDIS_OK) {
        fprintf(stderr, "error: ofdis_create failed with status %d for %dx%d frames\n", rc, w, h);
        return 1;
      }
      ofdis_set_graph_mode(ctx, 1);
      ctx_w = w;
      ctx_h = h;
    }
    const int slots = two_way ? 2 * n : n;  // two-way: forward slots [0, n), backward slots [n, 2n)
    const int kch = nop == 2 ? 3 : 1;     // --kitti: uint16 values per pixel
    if (kitti) kflows.resize((size_t)slots * w * h * kch);
    else flows.resize((size_t)slots * w * h * nop);
    int rc;
    if (two_way && seq) {
      rc = ofdis_upload_sequence_bidir_u8(ctx, 0, n, frames.data(), w, h, OFDIS_MEM_HOST);
    } else if (two_way) {
      rc = ofdis_upload_frames_u8(ctx, 0, 2 * n, frames.data(), w, h, OFDIS_MEM_HOST);
      if (rc == OFDIS_OK) rc = ofdis_set_swapped_slots(ctx, 0, n, 0);
      if (rc == OFDIS_OK) rc = ofdis_set_swapped_slots(ctx, n, 2 * n, 1);
    } else {
      rc = seq ? ofdis_upload_sequence_u8(ctx, 0, n, frames.data(), w, h, OFDIS_MEM_HOST)
               : ofdis_upload_frames_u8(ctx, 0, n, frames.data(), w, h, OFDIS_MEM_HOST);
    }
    // warm start: the context still holds the previous pair's flow (same size, so it was not recreated)
    const bool from_prev = warm && j0 > 0 && jobs[j0].a == jobs[j0 - 1].b;
    if (rc == OFDIS_OK && from_prev) rc = ofdis_set_initflow_from_result(ctx, 0, 1, 0, w, h);
    warm_pairs += from_prev ? 1 : 0;
    if (rc == OFDIS_OK) rc = ofdis_run(ctx, slots, from_prev ? 1 : 0);
    if (rc == OFDIS_OK)
      rc = kitti ? ofdis_get_flow_fullres_encoded(ctx, 0, slots, OFDIS_ENC_KITTI, kflows.data(), w, h, OFDIS_MEM_HOST)
                 : ofdis_get_flow_fullres(ctx, 0, slots, flows.data(), w, h, OFDIS_MEM_HOST);
    if (rc == OFDIS_OK && color) {
      colors.resize((size_t)slots * w * h * 3);
      rc = ofdis_flow_color_fullres(ctx, 0, slots, colors.data(), nullptr, color_max, w, h, OFDIS_MEM_HOST);
    }
    if (rc == OFDIS_OK && bidir) {
      masks.resize((size_t)n * w * h);
      rc = ofdis_consistency_fullres(ctx, 0, n, n, masks.data(), nullptr, nop == 2 ? 0.01f : 0.0f,
                                     nop == 2 ? 0.5f : 1.0f, w, h, OFDIS_MEM_HOST);
    }
    const size_t hwc = (size_t)w * h * nochannels;
    if (rc == OFDIS_OK && interp_arg) {
      // image1 / image2 of pair k: frames k and k + 1 of a clip, or the k-th pair of the pairs layout
      interp.resize((size_t)n * hwc);
      rc = ofdis_interpolate_fullres(ctx, 0, n, n, frames.data(), frames.data() + hwc, seq ? hwc : 2 * hwc, interp_t,
                                     nop == 2 ? 0.01f : 0.0f, nop == 2 ? 0.5f : 1.0f, interp.data(), nullptr, w, h,
                                     OFDIS_MEM_HOST);
    }
    if (rc == OFDIS_OK && gm_model) {
      // image2 of pair k: frame k + 1 of a clip, or the second image of the k-th pair
      const size_t np = (size_t)n * w * h;
      gm_models.resize((size_t)9 * n);
      gm_stats.resize(n);
      gm_mask.resize(np);
      gm_res.resize(2 * np);
      gm_reg.resize((size_t)n * hwc);
      ofdis_motion_params mp;
      memset(&mp, 0, sizeof(mp));
      mp.model = gm_model;
      mp.step = 8;
      mp.fb_check = bidir ? 1 : 0;
      mp.alpha = 0.01f;
      mp.beta = 0.5f;
      mp.hypotheses = 1024;
      mp.threshold = 1.0f;
      mp.refine = 3;
      mp.seed = 0;
      rc = ofdis_global_motion_fullres(ctx, 0, n, n, &mp, frames.data() + hwc, seq ? hwc : 2 * hwc, gm_models.data(),
                                       gm_stats.data(), gm_mask.data(), gm_res.data(), gm_reg.data(), w, h,
                                       OFDIS_MEM_HOST);
    }
    size_t dcount[6] = {0, 0, 0, 0, 0, 0};  // statuses 0..4, filled
    if (rc == OFDIS_OK && disp_on) {
      const size_t np = (size_t)n * w * h;
      ddisp.resize(np);
      dstatus.resize(np);
      ddepth.resize(camera_arg ? np : 0);
      dxyz.resize(camera_arg ? 3 * np : 0);
      rc = ofdis_disparity_fullres(ctx, 0, n, n, &dfilt, camera_arg ? &dcam : nullptr, ddisp.data(), dstatus.data(),
                                   camera_arg ? ddepth.data() : nullptr, camera_arg ? dxyz.data() : nullptr, w, h,
                                   OFDIS_MEM_HOST);
      for (size_t i = 0; i < np && rc == OFDIS_OK; ++i) {
        dcount[dstatus[i] < 5 ? dstatus[i] : 0] += 1;
        dcount[5] += dstatus[i] != 0 && !std::isnan(ddisp[i]);
      }
    }
    // --tracks: runs of pairs that continue each other; a run that does not continue the previous pair begins a clip
    for (int k0 = 0, k1; k0 < n && tracks_file && rc == OFDIS_OK; k0 = k1) {
      for (k1 = k0 + 1; k1 < n && jobs[j0 + k1].a == jobs[j0 + k1 - 1].b;) ++k1;
      const size_t fs = seq ? hwc : 2 * hwc;  // image1 of pair k at k * fs, its image2 one frame later
      const uint8_t* im1 = frames.data() + (size_t)k0 * fs;
      const uint8_t* im2 = im1 + hwc;
      ofdis_track_params tp;
      tp.spacing = 8;
      tp.capacity = 4 * ((w + 7) / 8) * ((h + 7) / 8);
      tp.alpha = nop == 2 ? 0.01f : 0.0f;
      tp.beta = nop == 2 ? 0.5f : 1.0f;
      tp.mb_alpha = 0.01f;
      tp.mb_beta = 0.002f;
      tp.min_eig = 25.0f;
      tpoints.resize((size_t)n * tp.capacity);
      tcounts.resize(n);
      if (j0 + k0 == 0 || jobs[j0 + k0].a != jobs[j0 + k0 - 1].b) {
        end_clip();
        rc = fisher_rc;
        ++tclip;
        tframe = 0;
        if (rc == OFDIS_OK)
          rc = traj_stage ? ofdis_traj_begin(ctx, &tp, &trp, im1, tpoints.data(), tcounts.data(), w, h, OFDIS_MEM_HOST)
                          : ofdis_track_begin(ctx, &tp, im1, tpoints.data(), tcounts.data(), w, h, OFDIS_MEM_HOST);
        if (rc == OFDIS_OK && fisher_file) {
          rc = ofdis_fisher_begin(ctx, &fbook.cb);
          fisher_live = rc == OFDIS_OK;
        }
        if (rc == OFDIS_OK) write_tracks(tpoints.data(), tcounts[0]);
      }
      if (rc == OFDIS_OK && traj_stage && !desc_file) {  // --fisher alone: the descriptors stay on the device
        tndesc.resize(k1 - k0);
        rc = ofdis_traj_advance_fisher(ctx, k0, k1, n + k0, im2, fs,
                                       gm_model ? gm_models.data() + (size_t)9 * k0 : nullptr, tpoints.data(),
                                       tcounts.data(), tndesc.data(), w, h, OFDIS_MEM_HOST);
      } else if (rc == OFDIS_OK && desc_file) {
        const size_t bound = (size_t)tp.capacity * ((k1 - k0 + 2 * trp.L - 2) / trp.L);
        trec.resize(bound);
        tdesc.resize(bound * tdim);
        tndesc.resize(k1 - k0);
        rc = ofdis_traj_advance(ctx, k0, k1, n + k0, im2, fs, gm_model ? gm_models.data() + (size_t)9 * k0 : nullptr,
                                tpoints.data(), tcounts.data(), trec.data(), tdesc.data(), tndesc.data(), w, h,
                                OFDIS_MEM_HOST);
        int total = 0;
        for (int k = 0; k < k1 - k0 && rc == OFDIS_OK; ++k) total += tndesc[k];
        if (rc == OFDIS_OK) write_desc(total);
        if (rc == OFDIS_OK && fisher_file) rc = ofdis_fisher_push(ctx, tdesc.data(), total, OFDIS_MEM_HOST);
      } else if (rc == OFDIS_OK) {
        rc = ofdis_track_advance(ctx, k0, k1, n + k0, im2, fs, tpoints.data(), tcounts.data(), w, h, OFDIS_MEM_HOST);
      }
      for (int k = 0; k < k1 - k0 && rc == OFDIS_OK; ++k) write_tracks(tpoints.data() + (size_t)k * tp.capacity, tcounts[k]);
    }
    // --stabilize: the runs of --tracks; a clip begins on its first image1, every run pushes its image2 frames with
    // their --global-motion models
    for (int k0 = 0, k1; k0 < n && stab_file && rc == OFDIS_OK; k0 = k1) {
      for (k1 = k0 + 1; k1 < n && jobs[j0 + k1].a == jobs[j0 + k1 - 1].b;) ++k1;
      const size_t fs = seq ? hwc : 2 * hwc;  // image1 of pair k at k * fs, its image2 one frame later
      const uint8_t* im1 = frames.data() + (size_t)k0 * fs;
      if (j0 + k0 == 0 || jobs[j0 + k0].a != jobs[j0 + k0 - 1].b) {
        rc = stab_end();
        if (rc == OFDIS_OK) rc = ofdis_stab_begin(ctx, &stp, stab_wts.data(), im1, w, h, OFDIS_MEM_HOST);
        if (rc == OFDIS_OK) {
          stab_live = true;
          ++sclip;
          sw = w;
          sh = h;
        }
      }
      if (rc != OFDIS_OK) break;
      sbuf.resize((size_t)(k1 - k0) * hwc);
      sinfo.resize(k1 - k0);
      int count = 0;
      rc = ofdis_stab_push(ctx, k1 - k0, gm_models.data() + (size_t)9 * k0, im1 + hwc, fs, sbuf.data(), sinfo.data(),
                           &count, OFDIS_MEM_HOST);
      if (rc == OFDIS_OK) write_stab(count);
    }
    if (rc == OFDIS_OK) rc = ofdis_sync(ctx);
    if (rc == OFDIS_OK && gtlist) {
      gt_batch.resize((size_t)n * w * h * nop);
      for (int k = 0; k < n; ++k) {
        string err;
        if (!read_gt_file(gts[j0 + k].c_str(), w, h, nop, gt_one, err)) {
          fprintf(stderr, "error: %s: %s\n", gts[j0 + k].c_str(), err.c_str());
          ofdis_destroy(ctx);
          return 1;
        }
        memcpy(gt_batch.data() + (size_t)k * w * h * nop, gt_one.data(), sizeof(float) * gt_one.size());
      }
      eval_pairs.resize((size_t)n * nclasses);
      rc = ofdis_flow_error_fullres(ctx, 0, n, gt_batch.data(), bidir ? masks.data() : nullptr, nclasses,
                                    eval_pairs.data(), nullptr, w, h, OFDIS_MEM_HOST);
      for (int k = 0; k < n && rc == OFDIS_OK; ++k)
        for (int c = 0; c < nclasses; ++c) {
          add_stats(eval_total[0], eval_pairs[(size_t)k * nclasses + c]);
          if (bidir) add_stats(eval_total[1 + c], eval_pairs[(size_t)k * nclasses + c]);
        }
    }
    if (rc == OFDIS_OK && sf_list) {
      const size_t pix = (size_t)w * h;
      // positive disparities: the readers return this library's stereo convention, -d
      auto load = [&](const string& path, int fnop, float sign, float* dst) {
        string err;
        if (!read_gt_file(path.c_str(), w, h, fnop, gt_one, err)) {
          fprintf(stderr, "error: %s: %s\n", path.c_str(), err.c_str());
          return false;
        }
        for (size_t i = 0; i < gt_one.size(); ++i) dst[i] = sign * gt_one[i];
        return true;
      };
      sf_d0.resize(n * pix);
      sf_d1.resize(n * pix);
      sf_w.resize(n * pix);
      sf_m.resize(camera_arg ? 3 * n * pix : 0);
      bool ok = true;
      for (int k = 0; k < n && ok; ++k)
        ok = load(sf_files[2 * (j0 + k)], 1, -1.0f, &sf_d0[k * pix]) && load(sf_files[2 * (j0 + k) + 1], 1, -1.0f, &sf_d1[k * pix]);
      if (sf_gtlist) {
        sf_g0.resize(n * pix);
        sf_g1.resize(n * pix);
        sf_gf.resize(2 * n * pix);
        for (int k = 0; k < n && ok; ++k)
          ok = load(sf_gts[3 * (j0 + k)], 1, -1.0f, &sf_g0[k * pix]) && load(sf_gts[3 * (j0 + k) + 1], 1, -1.0f, &sf_g1[k * pix]) &&
               load(sf_gts[3 * (j0 + k) + 2], 2, 1.0f, &sf_gf[2 * k * pix]);
        sf_pairs.resize((size_t)n * nclasses);
      }
      if (!ok) {
        ofdis_destroy(ctx);
        return 1;
      }
      const ofdis_sf_gt sgt{sf_g0.data(), sf_g1.data(), sf_gf.data()};
      rc = ofdis_scene_flow_fullres(ctx, 0, n, sf_d0.data(), sf_d1.data(), pix, 1.0f, camera_arg ? &dcam : nullptr,
                                    sf_w.data(), nullptr, camera_arg ? sf_m.data() : nullptr, sf_gtlist ? &sgt : nullptr,
                                    bidir ? masks.data() : nullptr, nclasses, sf_gtlist ? sf_pairs.data() : nullptr, w, h,
                                    OFDIS_MEM_HOST);
      for (int k = 0; k < n && rc == OFDIS_OK && sf_gtlist; ++k) {
        ofdis_sf_stats all;
        memset(&all, 0, sizeof(all));
        for (int c = 0; c < nclasses; ++c) {
          add_sf_stats(all, sf_pairs[(size_t)k * nclasses + c]);
          add_sf_stats(sf_total[1 + c], sf_pairs[(size_t)k * nclasses + c]);
        }
        add_sf_stats(sf_total[0], all);
        if (verbosity > 0) print_sfeval(jobs[j0 + k].out.c_str(), 0, all);
      }
      for (int k = 0; k < n && rc == OFDIS_OK; ++k) {
        const float* d = &sf_w[k * pix];
        if (kitti) {
          vector<uint16_t> enc(pix);
          for (size_t i = 0; i < pix; ++i)  // NaN fails d >= 0 and is written as 0
            enc[i] = d[i] >= 0.0f ? (uint16_t)fminf(fmaxf(d[i] * 256.0f, 1.0f), 65535.0f) : (uint16_t)0;
          save_png(enc.data(), w, h, 1, 16, with_suffix(jobs[j0 + k].out, "_disp1").c_str());
        } else {
          ImageF f;  // SavePFMFile writes -value: the positive disparity goes in as -d
          f.w = w; f.h = h; f.c = 1;
          f.px.resize(pix);
          for (size_t i = 0; i < pix; ++i) f.px[i] = -d[i];
          SavePFMFile(f, with_suffix(jobs[j0 + k].out, "_disp1", ".pfm").c_str());
        }
        if (camera_arg) save_pfm3(&sf_m[3 * k * pix], w, h, with_suffix(jobs[j0 + k].out, "_sceneflow", ".pfm").c_str());
      }
      if (rc == OFDIS_OK && odo_dir) {
        ofdis_egomotion_params ep;
        memset(&ep, 0, sizeof(ep));
        ep.step = 8;
        ep.fb_check = bidir ? 1 : 0;
        ep.alpha = 0.01f;
        ep.beta = 0.5f;
        ep.edge_diff = 1.0f;
        ep.hypotheses = 1024;
        ep.threshold = 1.0f;
        ep.refine = 5;
        ep.seed = 0;
        odo_pose.resize((size_t)12 * n);
        odo_stats.resize(n);
        odo_mask.resize(n * pix);
        odo_om.resize(3 * n * pix);
        rc = ofdis_egomotion_fullres(ctx, 0, n, n, &ep, sf_d0.data(), sf_d1.data(), pix, &dcam, odo_pose.data(),
                                     odo_stats.data(), odo_mask.data(), nullptr, odo_om.data(), w, h, OFDIS_MEM_HOST);
        for (int k = 0; k < n && rc == OFDIS_OK; ++k) {
          const int c = odo_clip[j0 + k], fr = odo_frame[j0 + k];
          const ofdis_motion_stats& st = odo_stats[k];
          const double* P = odo_pose.data() + (size_t)12 * k;
          fprintf(odo_file, "%d %d %d %d %d %d", c, fr, st.status, st.n_corr, st.ransac_inliers, st.n_inliers);
          for (int i = 0; i < 12; ++i) fprintf(odo_file, " %.17g", P[i]);
          fprintf(odo_file, "\n");
          odo_rel[c].insert(odo_rel[c].end(), P, P + 12);
          save_mask_pgm(odo_mask.data() + k * pix, w, h, with_suffix(jobs[j0 + k].out, "_objects", ".pgm").c_str());
          save_pfm3(&odo_om[3 * k * pix], w, h, with_suffix(jobs[j0 + k].out, "_objmotion", ".pfm").c_str());
          if (!odo_gtlist) continue;
          double te, re;
          pose_error(&odo_gt[c][(size_t)12 * fr], &odo_gt[c][(size_t)12 * (fr + 1)], P, &te, &re);
          odo_terr += te;
          odo_rerr += re;
          ++odo_eval;
          if (verbosity > 0) printf("ODOEVAL %d %d %.9g %.9g\n", c, fr, te, re);
        }
      }
      // --fuse: the runs of one clip within the batch; image1 of pair k at k * fs, its image2 one frame later
      const size_t fs = seq ? hwc : 2 * hwc;
      for (int k0 = 0, k1; k0 < n && rc == OFDIS_OK && fuse_arg; k0 = k1) {
        const int c = odo_clip[j0 + k0];
        for (k1 = k0 + 1; k1 < n && odo_clip[j0 + k1] == c;) ++k1;
        if (odo_frame[j0 + k0] == 0) {
          static const double kIdentity[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
          memcpy(fuse_T, kIdentity, sizeof(fuse_T));
          fuse_frames = 0;
          rc = ofdis_fuse_begin(ctx, &fuse_p);
          if (rc != OFDIS_OK) break;
        }
        fuse_poses.resize((size_t)12 * (k1 - k0 + 1));
        for (int k = k0; k < k1; ++k) {
          memcpy(&fuse_poses[(size_t)12 * (k - k0)], fuse_T, sizeof(fuse_T));
          chain_pose(fuse_T, odo_pose.data() + (size_t)12 * k);
        }
        memcpy(&fuse_poses[(size_t)12 * (k1 - k0)], fuse_T, sizeof(fuse_T));
        rc = ofdis_fuse_push(ctx, k1 - k0, &sf_d0[k0 * pix], pix, fuse_poses.data(), &dcam, INFINITY,
                             frames.data() + (size_t)k0 * fs, fs, w, h, OFDIS_MEM_HOST);
        fuse_frames += k1 - k0;
        if (rc != OFDIS_OK || (j0 + k1 < (int)jobs.size() && odo_clip[j0 + k1] == c)) continue;
        // the clip ends with this run: its last image2, then the surface
        rc = ofdis_fuse_push(ctx, 1, &sf_d1[(k1 - 1) * pix], pix, &fuse_poses[(size_t)12 * (k1 - k0)], &dcam, INFINITY,
                             frames.data() + (size_t)(k1 - 1) * fs + hwc, fs, w, h, OFDIS_MEM_HOST);
        ++fuse_frames;
        long count = 0;
        if (rc == OFDIS_OK) rc = ofdis_fuse_extract(ctx, 1.0f, nullptr, 0, &count, OFDIS_MEM_HOST);
        if (rc != OFDIS_OK) break;
        fuse_pts.resize(count);
        rc = ofdis_fuse_extract(ctx, 1.0f, fuse_pts.data(), count, &count, OFDIS_MEM_HOST);
        if (rc != OFDIS_OK) break;
        char name[32];
        snprintf(name, sizeof(name), "/fused_%04d.ply", c);
        string path = string(odo_dir) + name;
        if (!write_fused_ply(path, fuse_pts.data(), count, nochannels, false, nullptr, 0)) {
          fprintf(stderr, "error: cannot write %s\n", path.c_str());
          ofdis_destroy(ctx);
          return 1;
        }
        if (verbosity > 0) printf("FUSE clip %d frames %d points %ld\n", c, fuse_frames, count);
        if (!fuse_mesh) continue;
        // the mesh's vertices are the points just extracted: only the faces come back
        long nv = 0, nf = 0;
        rc = ofdis_fuse_mesh(ctx, 1.0f, nullptr, 0, &nv, nullptr, 0, &nf, OFDIS_MEM_HOST);
        if (rc != OFDIS_OK) break;
        fuse_faces.resize((size_t)3 * nf);
        rc = ofdis_fuse_mesh(ctx, 1.0f, nullptr, 0, &nv, fuse_faces.data(), nf, &nf, OFDIS_MEM_HOST);
        if (rc != OFDIS_OK) break;
        snprintf(name, sizeof(name), "/fused_%04d_mesh.ply", c);
        path = string(odo_dir) + name;
        if (!write_fused_ply(path, fuse_pts.data(), count, nochannels, true, fuse_faces.data(), nf)) {
          fprintf(stderr, "error: cannot write %s\n", path.c_str());
          ofdis_destroy(ctx);
          return 1;
        }
        if (verbosity > 0) printf("MESH clip %d vertices %ld faces %ld\n", c, nv, nf);
      }
    }
    if (rc != OFDIS_OK) {
      fprintf(stderr, "error: %s\n", ofdis_last_error(ctx));
      ofdis_destroy(ctx);
      return 1;
    }
    for (int k = 0; k < n && kitti; ++k) {
      save_png(kflows.data() + (size_t)k * w * h * kch, w, h, kch, 16, jobs[j0 + k].out.c_str());
      if (bidir) {
        save_png(kflows.data() + (size_t)(n + k) * w * h * kch, w, h, kch, 16,
                 with_suffix(jobs[j0 + k].out, "_bw").c_str());
        save_mask_pgm(masks.data() + (size_t)k * w * h, w, h, with_suffix(jobs[j0 + k].out, "_occ", ".pgm").c_str());
      }
    }
    for (int k = 0; k < n && color; ++k) {
      save_png(colors.data() + (size_t)k * w * h * 3, w, h, 3, 8, with_suffix(jobs[j0 + k].out, "_color", ".png").c_str());
      if (bidir)
        save_png(colors.data() + (size_t)(n + k) * w * h * 3, w, h, 3, 8,
                 with_suffix(jobs[j0 + k].out, "_bw_color", ".png").c_str());
    }
    for (int k = 0; k < n && interp_arg; ++k) {
      const uint8_t* im = interp.data() + (size_t)k * hwc;
      if (nochannels == 3) {  // the decoder's BGR -> RGB
        interp_png.resize(hwc);
        for (size_t p = 0; p < hwc; p += 3) {
          interp_png[p] = im[p + 2];
          interp_png[p + 1] = im[p + 1];
          interp_png[p + 2] = im[p];
        }
        im = interp_png.data();
      }
      save_png(im, w, h, nochannels, 8, with_suffix(jobs[j0 + k].out, "_interp", ".png").c_str());
    }
    for (int k = 0; k < n && gm_model; ++k) {
      const string& o = jobs[j0 + k].out;
      fprintf(gm_file, "%s", with_suffix(o, "", "").c_str());
      for (int i = 0; i < 9; ++i) fprintf(gm_file, " %.17g", gm_models[(size_t)9 * k + i]);
      fprintf(gm_file, " %d %d %d\n", gm_stats[k].status, gm_stats[k].n_corr, gm_stats[k].n_inliers);
      const float* r = gm_res.data() + (size_t)2 * k * w * h;
      if (kitti) {  // the encoding of OFDIS_ENC_KITTI (flow)
        vector<uint16_t> enc((size_t)3 * w * h);
        for (size_t i = 0; i < (size_t)w * h; ++i) {
          const float u = r[2 * i], v = r[2 * i + 1];
          const bool valid = !std::isnan(u) && !std::isnan(v);
          enc[3 * i] = valid ? (uint16_t)fminf(fmaxf(u * 64.0f + 32768.0f, 0.0f), 65535.0f) : (uint16_t)0;
          enc[3 * i + 1] = valid ? (uint16_t)fminf(fmaxf(v * 64.0f + 32768.0f, 0.0f), 65535.0f) : (uint16_t)0;
          enc[3 * i + 2] = valid ? 1 : 0;
        }
        save_png(enc.data(), w, h, 3, 16, with_suffix(o, "_residual").c_str());
      } else {
        ImageF f;
        f.w = w; f.h = h; f.c = 2;
        f.px.assign(r, r + (size_t)2 * w * h);
        SaveFlowFile(f, with_suffix(o, "_residual").c_str());
      }
      save_mask_pgm(gm_mask.data() + (size_t)k * w * h, w, h, with_suffix(o, "_moving", ".pgm").c_str());
      const uint8_t* im = gm_reg.data() + (size_t)k * hwc;
      if (nochannels == 3) {  // the decoder's BGR -> RGB
        gm_png.resize(hwc);
        for (size_t q = 0; q < hwc; q += 3) {
          gm_png[q] = im[q + 2];
          gm_png[q + 1] = im[q + 1];
          gm_png[q + 2] = im[q];
        }
        im = gm_png.data();
      }
      save_png(im, w, h, nochannels, 8, with_suffix(o, "_registered", ".png").c_str());
    }
    for (int k = 0; k < n && disp_on; ++k) {
      const size_t o = (size_t)k * w * h;
      if (kitti) {
        vector<uint16_t> enc((size_t)w * h);
        for (size_t i = 0; i < enc.size(); ++i) {
          const float d = ddisp[o + i];  // NaN fails d >= 0 and is written as 0
          enc[i] = d >= 0.0f ? (uint16_t)fminf(fmaxf(d * 256.0f, 1.0f), 65535.0f) : (uint16_t)0;
        }
        save_png(enc.data(), w, h, 1, 16, with_suffix(jobs[j0 + k].out, "_filtered").c_str());
      } else {
        ImageF f;  // SavePFMFile writes -value: the positive disparity goes in as -d, the sign of <stem><ext>
        f.w = w; f.h = h; f.c = 1;
        f.px.resize((size_t)w * h);
        for (size_t i = 0; i < f.px.size(); ++i) f.px[i] = -ddisp[o + i];
        SavePFMFile(f, with_suffix(jobs[j0 + k].out, "_filtered").c_str());
      }
      if (!camera_arg) continue;
      ImageF z;
      z.w = w; z.h = h; z.c = 1;
      z.px.resize((size_t)w * h);
      for (size_t i = 0; i < z.px.size(); ++i) z.px[i] = -ddepth[o + i];
      SavePFMFile(z, with_suffix(jobs[j0 + k].out, "_depth", ".pfm").c_str());
      // image1 of pair k: frame k of a clip, or the first image of the k-th pair
      const uint8_t* im1 = frames.data() + (size_t)k * (seq ? hwc : 2 * hwc);
      size_t npts = 0;
      dply.clear();
      for (size_t i = 0; i < (size_t)w * h; ++i) {
        if (!std::isfinite(ddepth[o + i])) continue;
        const float* q = dxyz.data() + (o + i) * 3;
        const uint8_t* c = im1 + i * nochannels;
        const uint8_t rgb[3] = {nochannels == 3 ? c[2] : c[0], c[nochannels == 3 ? 1 : 0], c[0]};  // the decoder's BGR
        const uint8_t* qb = reinterpret_cast<const uint8_t*>(q);
        dply.insert(dply.end(), qb, qb + 12);
        dply.insert(dply.end(), rgb, rgb + 3);
        ++npts;
      }
      const string ply = with_suffix(jobs[j0 + k].out, "", ".ply");
      FILE* pf = fopen(ply.c_str(), "wb");
      if (!pf) {
        cout << "WriteFile: could not open file" << endl;
        continue;
      }
      fprintf(pf, "ply\nformat binary_little_endian 1.0\nelement vertex %zu\nproperty float x\nproperty float y\n"
                  "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n", npts);
      if (fwrite(dply.data(), 1, dply.size(), pf) != dply.size()) cout << "WriteFile: problem writing data" << endl;
      fclose(pf);
    }
    if (verbosity > 0 && disp_on)
      printf("DISP pairs %d valid %zu inconsistent %zu leaves %zu range %zu speckle %zu filled %zu\n", n, dcount[0],
             dcount[1], dcount[2], dcount[3], dcount[4], dcount[5]);
    ImageF out;
    out.w = w; out.h = h; out.c = nop;
    for (int k = 0; k < n && !kitti; ++k) {
      out.px.assign(flows.begin() + (size_t)k * w * h * nop, flows.begin() + (size_t)(k + 1) * w * h * nop);
      if (SELECTMODE == 1) SaveFlowFile(out, jobs[j0 + k].out.c_str());
      else SavePFMFile(out, jobs[j0 + k].out.c_str());
      if (!bidir) continue;
      out.px.assign(flows.begin() + (size_t)(n + k) * w * h * nop, flows.begin() + (size_t)(n + k + 1) * w * h * nop);
      const string bw = with_suffix(jobs[j0 + k].out, "_bw");
      if (SELECTMODE == 1) SaveFlowFile(out, bw.c_str());
      else SavePFMFile(out, bw.c_str());
      save_mask_pgm(masks.data() + (size_t)k * w * h, w, h, with_suffix(jobs[j0 + k].out, "_occ", ".pgm").c_str());
    }
    j0 += n;
    done += n;
  }
  end_clip();
  if (fisher_rc != OFDIS_OK || stab_end() != OFDIS_OK) {
    fprintf(stderr, "error: %s\n", ofdis_last_error(ctx));
    ofdis_destroy(ctx);
    return 1;
  }
  if (ctx) ofdis_destroy(ctx);
  if (stab_file && fclose(stab_file) != 0) {
    fprintf(stderr, "error: cannot write %s\n", stab_txt.c_str());
    return 1;
  }
  if (tracks_file && fclose(tracks_file) != 0) {
    fprintf(stderr, "error: cannot write %s\n", tracks_path);
    return 1;
  }
  if (desc_file && fclose(desc_file) != 0) {
    fprintf(stderr, "error: cannot write %s\n", desc_path);
    return 1;
  }
  if (fisher_file && fclose(fisher_file) != 0) {
    fprintf(stderr, "error: cannot write %s\n", fisher_arg[1]);
    return 1;
  }
  if (gm_file && fclose(gm_file) != 0) {
    fprintf(stderr, "error: cannot write %s\n", gm_arg[1]);
    return 1;
  }
  if (odo_file && fclose(odo_file) != 0) {
    fprintf(stderr, "error: cannot write %s/odometry.txt\n", odo_dir);
    return 1;
  }
  for (size_t c = 0; c < odo_rel.size(); ++c) {
    char name[32];
    snprintf(name, sizeof(name), "/poses_%04zu.txt", c);
    const string path = string(odo_dir) + name;
    FILE* f = fopen(path.c_str(), "w");
    double T[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    for (size_t k = 0; f && k <= odo_rel[c].size() / 12; ++k) {
      if (k > 0) chain_pose(T, &odo_rel[c][12 * (k - 1)]);
      for (int i = 0; i < 12; ++i) fprintf(f, i ? " %.17g" : "%.17g", T[i]);
      fprintf(f, "\n");
    }
    if (!f || fclose(f) != 0) {
      fprintf(stderr, "error: cannot write %s\n", path.c_str());
      return 1;
    }
  }
  if (verbosity > 0) printf("TIME (%zu pairs, load + flow + save) (ms): %3g\n", done, elapsed_ms(tv));
  if (verbosity > 0 && seq_pairs) printf("SEQUENCE (%zu of %zu pairs from %zu decoded frames)\n", seq_pairs, done, seq_decoded);
  if (verbosity > 0 && warm) printf("WARM START (%zu of %zu pairs from the previous pair's flow)\n", warm_pairs, done);
  if (verbosity > 0 && tracks_path)
    printf("TRACKS clips %d frames %zu seeded %lld leaves %lld inconsistent %lld boundary %lld dropped %lld\n", tclip + 1,
           tframes, ttotal.seeded, ttotal.ended_leaves, ttotal.ended_inconsistent, ttotal.ended_boundary, ttotal.dropped);
  if (verbosity > 0 && desc_path)
    printf("DESCRIPTORS clips %d emitted %lld static %lld erratic %lld jump %lld camera %lld\n", tclip + 1,
           dtotal.emitted, dtotal.rejected_static, dtotal.rejected_erratic, dtotal.rejected_jump, dtotal.rejected_camera);
  if (verbosity > 0 && fisher_arg[0]) {
    printf("FISHER clips %d descriptors %lld skipped", fclips, fpushed);
    for (int b = 0; b < fbook.cb.nblocks; ++b) printf(" %lld", fskipped[b]);
    printf("\n");
  }
  if (verbosity > 0 && gtlist) {
    static const char* const kClassNames[3] = {"consistent", "inconsistent", "leaves"};
    print_eval("", done, eval_total[0]);
    for (int c = 0; c < nclasses && bidir; ++c) print_eval(kClassNames[c], done, eval_total[1 + c]);
  }
  if (verbosity > 0 && odo_gtlist)
    printf("ODOEVAL (%zu pairs) t_err %.9g r_err %.9g\n", odo_eval, odo_eval ? odo_terr / odo_eval : 0.0,
           odo_eval ? odo_rerr / odo_eval : 0.0);
  if (verbosity > 0 && sf_gtlist) {
    static const char* const kClassNames[3] = {"consistent", "inconsistent", "leaves"};
    print_sfeval("", done, sf_total[0]);
    for (int c = 0; c < nclasses && bidir; ++c) print_sfeval(kClassNames[c], done, sf_total[1 + c]);
  }
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
