// Window geometry of the tiled forward (wn_enhance_u8_tiled).  The apply kernel, the gate epilogue, the per-pixel
// kernels of a pass (slot geometry, below) and the host planner all call these functions: this is the only place
// that knows the rule.
//
// Every output pixel of WaterNet depends on the input within kTileHalo pixels (the eight cmg convolutions have
// radii 3+2+1+0+3+2+1+1; the refiners need 6, the gate is per pixel).  An image is cut into balanced output tiles
// of at most tile_h x tile_w; tile (i, j) keeps rows [i*th, min(H, (i+1)*th)) and is computed from a window of
// win_h x win_w image pixels around it, clamped into the image.  All windows of a call have the same size, every
// window edge inside the image is at least kTileHalo pixels from the kept rectangle, and a window edge on the
// image border sees the same zero padding as the untiled forward: every kept pixel sees the operands it sees
// untiled (DESIGN.md "Tiled enhance").
#pragma once

#include <stdint.h>

#include <algorithm>
#include <vector>

namespace wn {

constexpr int kTileHalo = 13;

struct TileGeom {
  int H, W;          // image
  int th, tw;        // kept tile (balanced: <= the requested tile)
  int ny, nx;        // tiles per image column / row
  int win_h, win_w;  // window
};

// tile_h, tile_w >= 1 and H, W >= 1 (checked by the callers)
__host__ __device__ inline TileGeom tile_geom(int H, int W, int tile_h, int tile_w) {
  TileGeom g;
  g.H = H;
  g.W = W;
  g.ny = (H + tile_h - 1) / tile_h;
  g.nx = (W + tile_w - 1) / tile_w;
  g.th = (H + g.ny - 1) / g.ny;  // (ny - 1) * th < H: no tile is empty
  g.tw = (W + g.nx - 1) / g.nx;
  g.win_h = g.th + 2 * kTileHalo < H ? g.th + 2 * kTileHalo : H;
  g.win_w = g.tw + 2 * kTileHalo < W ? g.tw + 2 * kTileHalo : W;
  return g;
}

// window `win` of a call, numbered (image, tile row, tile column): its image, its origin and its kept rectangle
// [ky0, ky1) x [kx0, kx1), all in image coordinates
struct TileWindow {
  int img, ys, xs, ky0, ky1, kx0, kx1;
};

__host__ __device__ inline int tile_clamp(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

__host__ __device__ inline TileWindow tile_window(const TileGeom& g, long long win) {
  const long long per_image = (long long)g.ny * g.nx;
  TileWindow t;
  t.img = (int)(win / per_image);
  const int r = (int)(win - t.img * per_image);
  const int i = r / g.nx, j = r - i * g.nx;
  t.ky0 = i * g.th;
  t.kx0 = j * g.tw;
  t.ky1 = t.ky0 + g.th < g.H ? t.ky0 + g.th : g.H;
  t.kx1 = t.kx0 + g.tw < g.W ? t.kx0 + g.tw : g.W;
  t.ys = tile_clamp(t.ky0 - kTileHalo, 0, g.H - g.win_h);
  t.xs = tile_clamp(t.kx0 - kTileHalo, 0, g.W - g.win_w);
  return t;
}

// The windows whose extent contains image pixel (y, x): tile rows [i0, i1] x tile columns [j0, j1] of its image, the
// window numbering of tile_window (row-major).  Window i starts at ys(i) = clamp(i*th - kTileHalo, 0, H - win_h),
// which does not decrease with i, so the windows containing a row form one run: i1 is the last with ys(i) <= y, i0
// the first with ys(i) + win_h > y.  Every pixel lies in its own tile's window, so the run is never empty.  Tiles
// smaller than 2 * kTileHalo put a pixel in three or more windows per axis; when win_h == H every window contains it.
struct TileCover {
  int i0, i1, j0, j1;
};

__host__ __device__ inline void tile_cover_axis(int v, int size, int t, int count, int win, int* lo, int* hi) {
  *hi = v >= size - win ? count - 1 : (v + kTileHalo) / t < count - 1 ? (v + kTileHalo) / t : count - 1;
  const int first = v - win + 1;  // ys(i) >= first
  *lo = first <= 0 ? 0 : (first + kTileHalo + t - 1) / t;
}

__host__ __device__ inline TileCover tile_cover(const TileGeom& g, int y, int x) {
  TileCover c;
  tile_cover_axis(y, g.H, g.th, g.ny, g.win_h, &c.i0, &c.i1);
  tile_cover_axis(x, g.W, g.tw, g.nx, g.win_w, &c.j0, &c.j1);
  return c;
}

// windows per pass: as many as fit in max_pass_pixels (at least one, at most all of them and at most 65535, the
// grid limit of the per-window apply kernel)
__host__ __device__ inline long long tile_pass_windows(const TileGeom& g, int n, long long max_pass_pixels) {
  const long long total = (long long)n * g.ny * g.nx;
  long long p = max_pass_pixels / ((long long)g.win_h * g.win_w);
  if (p > total) p = total;
  if (p > 65535) p = 65535;
  return p < 1 ? 1 : p;
}

// ---- ragged batches (wn_enhance_u8_ragged): n images of their own sizes in one call ----
// Image i is cut into exactly the windows wn_enhance_u8_tiled would use for it alone (tile_geom / tile_window).  The
// windows of all images are sorted by shape and packed into passes; a pass runs as a batch of equally sized *slots*
// (the per-axis maximum of its windows), each window at its slot's top-left.  Slot pixels beyond a window's valid
// extent vh x vw are stored as zeros by every layer (the windowed apply kernel and the kEpiAct epilogues), so that
// each window sees the same zero padding as the tiled call (DESIGN.md "Ragged batches").
struct RaggedWindow {
  const uint8_t* rgb;      // the image, HWC uint8
  uint8_t* out_u8;         // its HWC uint8 output
  float* out_f32;          // its fp32 NCHW output, or null
  int img, H, W;           // image index and size
  int ys, xs;              // window origin in the image
  int vh, vw;              // valid extent: the window's size
  int ky0, ky1, kx0, kx1;  // kept rectangle, image coordinates
  int tile;                // the window's index within its image (tile_window numbering)
};
static_assert(sizeof(RaggedWindow) == 72, "RaggedWindow: engine.RAGGED_WINDOW_BYTES restates this size");

struct RaggedPass {
  long long first;  // first window (index into the sorted table)
  int count;        // windows
  int slot_h, slot_w;
};

// max_pass_pixels > 0; the caller has checked n, the sizes and the tile.  Windows go into *wins in pass order
// (shape sorted: taller first, then wider, then image and window order) with their pointers left null.  All windows
// of one image have one shape, so the stable sort keeps them contiguous and in ascending tile order.  A window
// joins the open pass unless that would break one of its limits: count x slot pixels <= max_pass_pixels, at most
// 65535 windows (the grid limit of the apply kernel), and masked padding at most a quarter of the slot pixels.
inline void ragged_plan(const int* hs, const int* ws, int n, int tile_h, int tile_w, long long max_pass_pixels,
                        std::vector<RaggedWindow>* wins, std::vector<RaggedPass>* passes) {
  wins->clear();
  passes->clear();
  for (int i = 0; i < n; i++) {
    const TileGeom g = tile_geom(hs[i], ws[i], tile_h, tile_w);
    for (long long k = 0; k < (long long)g.ny * g.nx; k++) {
      const TileWindow t = tile_window(g, k);
      RaggedWindow r = {};
      r.img = i;
      r.H = g.H;
      r.W = g.W;
      r.ys = t.ys;
      r.xs = t.xs;
      r.vh = g.win_h;
      r.vw = g.win_w;
      r.ky0 = t.ky0;
      r.ky1 = t.ky1;
      r.kx0 = t.kx0;
      r.kx1 = t.kx1;
      r.tile = (int)k;
      wins->push_back(r);
    }
  }
  std::stable_sort(wins->begin(), wins->end(), [](const RaggedWindow& a, const RaggedWindow& b) {
    return a.vh != b.vh ? a.vh > b.vh : a.vw > b.vw;
  });
  RaggedPass p = {0, 0, 0, 0};
  long long valid = 0;
  for (size_t k = 0; k < wins->size(); k++) {
    const RaggedWindow& w = (*wins)[k];
    if (p.count > 0) {
      const long long cnt = p.count + 1;
      const long long slot = (long long)(p.slot_h > w.vh ? p.slot_h : w.vh) * (p.slot_w > w.vw ? p.slot_w : w.vw);
      const long long v = valid + (long long)w.vh * w.vw;
      if (cnt <= 65535 && cnt * slot <= max_pass_pixels && 4 * (cnt * slot - v) <= cnt * slot) {
        p.count++;
        p.slot_h = p.slot_h > w.vh ? p.slot_h : w.vh;
        p.slot_w = p.slot_w > w.vw ? p.slot_w : w.vw;
        valid = v;
        continue;
      }
      passes->push_back(p);
    }
    p.first = (long long)k;
    p.count = 1;
    p.slot_h = w.vh;
    p.slot_w = w.vw;
    valid = (long long)w.vh * w.vw;
  }
  if (p.count > 0) passes->push_back(p);
}

// the pixels of a pass list's largest pass (its workspace is sized for that one)
inline long long largest_pass_pixels(const std::vector<RaggedPass>& passes) {
  long long px = 0;
  for (const RaggedPass& p : passes) px = std::max(px, (long long)p.count * p.slot_h * p.slot_w);
  return px;
}

// the passes of `total` slots of one grid geometry, slots [first, first + per_pass) each
inline std::vector<RaggedPass> grid_passes(long long total, long long per_pass, int slot_h, int slot_w) {
  std::vector<RaggedPass> passes;
  for (long long first = 0; first < total; first += per_pass)
    passes.push_back({first, (int)std::min(per_pass, total - first), slot_h, slot_w});
  return passes;
}

// ---- slot geometry: where pixel pix of slot s of a pass sits in its image ----
// A pass runs a batch of slots, each holding one window (or one whole image) at its top-left.  Every per-pixel kernel
// of a pass that reads or writes image coordinates (the operand packing, the kept-rectangle store, the backward's
// seed, input-gradient copy and fold) asks one of two geometries: GridGeom, window w0 + s of one tile_geom (an
// untiled call is the case tile = image size and w0 = 0: slot s is image s, kept everywhere), and TableGeom, window
// wins[w0 + s] of a ragged plan.  Each user pairs the geometry with its own per-image data.
struct SlotPixel {
  int img;          // the image
  int y, x;         // image coordinates
  bool valid;       // inside the slot's valid extent (slot pixels beyond it hold no image pixel)
  bool kept;        // valid and inside the window's kept rectangle
  size_t ihw, o;    // the image's plane size, and y * W + x
  TileGeom tiles;   // the windows its image is cut into (the backward's fold)
  long long k0;     // its image's tile k is window k0 + k of the pass's numbering
};

struct GridGeom {
  TileGeom tiles;
  long long w0;
  __host__ __device__ int slot_width() const { return tiles.win_w; }
  __host__ __device__ int slot_hw() const { return tiles.win_h * tiles.win_w; }
  // host: the slots of pass q, and the window table of its masked forward (FwdOpts::rwin; none for a grid)
  void set_pass(const RaggedPass& q) { w0 = q.first; }
  const RaggedWindow* rwin() const { return nullptr; }
  __device__ void origin(long long k, int* ys, int* xs) const {
    const TileWindow t = tile_window(tiles, k);
    *ys = t.ys;
    *xs = t.xs;
  }
  __device__ SlotPixel at(int s, int pix) const {
    const TileWindow t = tile_window(tiles, w0 + s);
    const int wy = pix / tiles.win_w;
    SlotPixel p;
    p.y = t.ys + wy;
    p.x = t.xs + (pix - wy * tiles.win_w);
    p.valid = true;
    p.kept = p.y >= t.ky0 && p.y < t.ky1 && p.x >= t.kx0 && p.x < t.kx1;
    p.img = t.img;
    p.ihw = (size_t)tiles.H * tiles.W;
    p.o = (size_t)p.y * tiles.W + p.x;
    p.tiles = tiles;
    p.k0 = (long long)t.img * tiles.ny * tiles.nx;
    return p;
  }
};

// the slots of an untiled call of n images of H x W: slot s is image s, whole
inline GridGeom whole_images(int H, int W) { return {tile_geom(H, W, H, W), 0}; }

// Slot s is window wins[w0 + s] at the top-left of a slot_h x slot_w slot; each image is cut into the windows of
// tile_geom(H, W, tile_h, tile_w), contiguous in the plan in ascending tile order (the callers of the fold check this
// on the host), so tile k of the image of plan window w is plan window w - wins[w].tile + k.
struct TableGeom {
  const RaggedWindow* wins;
  long long w0;
  int slot_h, slot_w;
  int tile_h, tile_w;
  __host__ __device__ int slot_width() const { return slot_w; }
  __host__ __device__ int slot_hw() const { return slot_h * slot_w; }
  void set_pass(const RaggedPass& q) {
    w0 = q.first;
    slot_h = q.slot_h;
    slot_w = q.slot_w;
  }
  const RaggedWindow* rwin() const { return wins + w0; }
  __device__ void origin(long long k, int* ys, int* xs) const {
    *ys = wins[k].ys;
    *xs = wins[k].xs;
  }
  __device__ SlotPixel at(int s, int pix) const {
    const long long me = w0 + s;
    const RaggedWindow& r = wins[me];
    const int wy = pix / slot_w, wx = pix - wy * slot_w;
    SlotPixel p;
    p.y = r.ys + wy;
    p.x = r.xs + wx;
    p.valid = wy < r.vh && wx < r.vw;
    p.kept = p.valid && p.y >= r.ky0 && p.y < r.ky1 && p.x >= r.kx0 && p.x < r.kx1;
    p.img = r.img;
    p.ihw = (size_t)r.H * r.W;
    p.o = (size_t)p.y * r.W + p.x;
    p.tiles = tile_geom(r.H, r.W, tile_h, tile_w);
    p.k0 = me - r.tile;
    return p;
  }
};

}  // namespace wn
