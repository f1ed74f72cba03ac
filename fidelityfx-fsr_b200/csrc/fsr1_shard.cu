// fsr1_shard.cu — row-slab sharding of the EASU+RCAS path across the GPUs of one box, with the EASU input halo
// moved by DIRECT NVLink stores into the neighbour's memory (SURVEY.md §8(e) "Alternative": P2P mapped slabs).
//
// The reference has no multi-GPU path (sample/src/DX12/FSRSample.cpp:901 is a comment); this is new.  One fsr1_shard
// per rank (= per GPU; ranks may be processes, attached through CUDA IPC handles, or live in one process, attached
// by pointer).  The OUTPUT image is cut into `world` row slabs; rank k owns input rows [k inH/world, (k+1) inH/world)
// and needs 2-3 more rows each side (the EASU footprint of its slab plus the one-row apron RCAS reads).
//
// Data plane per frame (no NCCL, no host round trip, no collective, and NO extra launch on the streams the big kernels use):
//   comm stream   halo_push_kernel, 2 x 8 one-warp CTAs on a HIGH-PRIORITY stream (a 32-thread CTA fits beside the six resident EASU
//   (high prio)   CTAs a halo-waiting launch puts on an SM and is dispatched ahead of pending RCAS CTAs): half of them copy my top rows into the upper neighbour's
//                 window (its bottom halo), the others my bottom rows into the lower neighbour's — 128-bit stores over NVLink,
//                 __threadfence_system, then a release store of the frame's sequence number into the neighbour's `ready` flag.
//   EASU stream   the EASU (or fused) kernel itself carries the hand-shake (HaloSync, fsr1_common.cuh): every CTA's thread 0
//                 acquires MY `ready` flags before the CTA's first load, the last CTA to finish release-stores the sequence
//                 number into the neighbours' `credit` flags ("your rows in my window may be overwritten").  Kernels without
//                 that hook (UNORM, fp32, direct) get the same protocol from two one-warp kernels around them.
//   two compute streams, whole frames in turn: RCAS of frame i overlaps EASU of frame i+1 exactly as on one GPU.
// Flow control is by sequence numbers in device memory, so it is independent of host timing on either side: a push
// for the q-th use of a slot waits for credit q-1, EASU of use q waits for ready q.  Every spin is bounded (a wall
// clock timeout sets an error word instead of hanging the GPU).
//
// Dynamic resolution (FSR1_SHARD_DYNAMIC, fsr1_shard_frame): every use of a slot may have its own render size rw x rh (the
// top-left of the input resource) and sharpness.  The frame's plan — owned / needed / window rows, the rows pushed to each
// neighbour and where they land in the neighbour's window — is a pure function of (rh, constants, world, rank), so both ends
// of a push compute the same destination rows without talking.  Each slot's window has room for the tallest window of any
// render height the shard accepts, on every rank (the arena layout is rank-independent).
// The protocol, and the credit sent by the EASU (or fused) kernel's last CTA, are those of a static shard.  Two kernels read my
// window during use q-1 of a slot: my EASU kernel, and my push, which copies my edge rows to BOTH neighbours in one launch and may
// still wait for one neighbour's credit after my EASU has finished and credited the other.  The credit covers the EASU's reads.
// My push's reads for use q-1 on the side of a neighbour are ordered before that neighbour's push for use q: they published the
// neighbour's ready q-1, which its EASU of use q-1 waited for, and the neighbour writes its rows for use q (and submits) only after
// its fsr1_shard_wait of use q-1.  Nothing orders them before the OTHER neighbour's push for use q, so that one must never write a
// row my push reads for use q-1 on the opposite side.  With one height for every use that always holds (neighbours write halo
// rows, my push reads owned rows).  With a height per use it does not by itself: at 8 ranks, a 100-row frame and then a 21-row
// one put rank 2's rows for the second frame on window rows rank 1's push up reads for the first.  So fsr1_shard_create marks,
// per rank, the window offsets the push to each side reads and the neighbour on each side writes, over the accepted heights from
// in_h downwards, and stops at the first height at which a row written from below would be a row read by the push up of some
// accepted height, or the mirror case (mark_push_rows); fsr1_shard_frame refuses every height below (FSR1_ERR_UNSUPPORTED).  In
// practice that is heights of a few rows per rank.  With that, the neighbour's push for use q waits for my credit q-1, so it never
// overwrites a row my EASU of use q-1 still reads, and it never writes a row my push of use q-1 may still read; my own rows for use q are
// written after fsr1_shard_wait of use q-1 (which follows my push); and every row EASU reads for use q (needed rows, all inside
// [owned(k-1).a, owned(k+1).b)) is written for use q, by me or by a neighbour, before ready q is released, so rows a previous frame
// left in the window are never read.
//
// Display output (fsr1_shard_create_post, fsr1_shard_post): every frame is fsr1_upscale_post with the shard's ops and the slot's
// description (frame, amount, tiles) instead of fsr1_upscale, so the slab is written once in the display format.  The fused post
// kernel and the tiled EASU before the RCAS post kernel carry HaloSync like their plain forms; nothing else about the protocol changes.
#include <new>
#include <string.h>
#include <vector>

#include "../../include/fsr1_b200.h"
#include "fsr1_common.cuh"

namespace {

using fsr1::bytes_per_pixel;
using fsr1::easu_out_format;
using fsr1::Rows;
using fsr1::spin_until;
using fsr1::st_release_sys;

constexpr uint32_t kFlagBytes = 4096;          // flags page at the start of the arena
constexpr uint32_t kMaxSlots = 128;

enum { kFromUp = 0, kFromDown = 1 };
// flag word index inside an arena's flags page
__host__ __device__ inline uint32_t ready_idx(uint32_t slot, int from) { return slot * 4 + from; }
__host__ __device__ inline uint32_t credit_idx(uint32_t slot, int from) { return slot * 4 + 2 + from; }
constexpr uint32_t kStatusIdx = kMaxSlots * 4;  // != 0: a spin timed out (value = 1 + which)
__host__ __device__ inline uint32_t counter_idx(uint32_t slot) { return kStatusIdx + 1 + slot; }  // CTAs of the slot's EASU that finished
__host__ __device__ inline uint32_t push_cnt_idx(uint32_t slot, int side) { return kStatusIdx + 1 + kMaxSlots + slot * 2 + side; }  // push parts done
constexpr int kPushParts = 8;  // one-warp CTAs per direction
constexpr uint32_t kTraceFrames = 256, kTraceWords = 8;  // fsr1_shard_trace: device timestamps of the last frames

struct PushSide {
  const uint4* src;        // my rows (local)
  uint4* dst;              // the neighbour's window rows (peer memory); nullptr = no neighbour on this side
  uint32_t n16;            // 16-byte units
  const uint32_t* credit;  // local: the neighbour has finished reading the previous use of this slot
  uint32_t* ready;         // peer: "your halo rows for use q are in place"
  uint32_t* parts_done;    // local: one-warp CTAs of this push that have finished
  unsigned long long* trace;  // optional: [3 + 2 side] first part started copying, [4 + 2 side] published
};

// kPushParts one-warp CTAs per direction (blockIdx.x / kPushParts = 0: up, 1: down), each moving 1/kPushParts of the rows.  32 threads
// and < 32 registers: such a CTA fits into what a halo-waiting EASU launch (6 CTAs per SM, launch_easu_h_tiled) or the fused kernel
// (6 per SM) leaves of an SM, so a push never waits for a big kernel to finish.  Stores over NVLink are fire-and-forget; two 16-byte loads per lane are kept in flight.  The last part to finish (counter in
// local memory) publishes the sequence number.
__global__ void __launch_bounds__(32) halo_push_kernel(const PushSide up, const PushSide down, const uint32_t q, uint32_t* status) {
  const int side = blockIdx.x / kPushParts, part = blockIdx.x - side * kPushParts;
  const PushSide s = side == 0 ? up : down;
  if (!s.dst) return;
  int ok = 1;
  if (threadIdx.x == 0) {
    ok = spin_until(s.credit, q - 1) ? 1 : 0;
    if (!ok) atomicExch(status, 1u + side);
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  if (s.trace && part == 0 && threadIdx.x == 0) s.trace[3 + 2 * side] = fsr1::global_ns();
  if (ok) {
    const uint32_t per = (s.n16 + kPushParts - 1) / kPushParts, first = part * per;
    const uint32_t end = first + per < s.n16 ? first + per : s.n16;
    const uint32_t t0 = first + threadIdx.x;
    uint32_t left = end > t0 ? (end - t0 + 31) / 32 : 0;  // 16-byte units this lane moves
    const uint4* src = s.src + t0;
    uint4* dst = s.dst + t0;
#pragma unroll 1
    for (; left >= 2; left -= 2, src += 64, dst += 64) {
      const uint4 a = src[0], b = src[32];
      dst[0] = a;
      dst[32] = b;
    }
    if (left) dst[0] = src[0];
    __threadfence_system();
  }
  __syncwarp();
  if (threadIdx.x == 0 && atomicAdd(s.parts_done, 1u) == kPushParts - 1) {  // last part (a timed-out push publishes nothing)
    atomicExch(s.parts_done, 0u);
    __threadfence_system();  // acquire side of the counter: the other parts' stores (fenced before their increment) precede the flag
    if (ok) st_release_sys(s.ready, q);
    if (s.trace) s.trace[4 + 2 * side] = fsr1::global_ns();
  }
}

__global__ void __launch_bounds__(32) halo_wait_kernel(const uint32_t* ready_up, const uint32_t* ready_down, const uint32_t q, uint32_t* status) {
  const uint32_t* f = threadIdx.x == 0 ? ready_up : (threadIdx.x == 1 ? ready_down : nullptr);
  if (f && !spin_until(f, q)) atomicExch(status, 3u + threadIdx.x);
}

__global__ void __launch_bounds__(32) credit_signal_kernel(uint32_t* credit_up, uint32_t* credit_down, const uint32_t q) {
  uint32_t* f = threadIdx.x == 0 ? credit_up : (threadIdx.x == 1 ? credit_down : nullptr);
  if (f) st_release_sys(f, q);
}

// the fsr1_shard_* bits of the create flags; the rest are FSR1_FLAG_* for the kernels
constexpr uint32_t kShardFlags = FSR1_SHARD_ONE_STREAM | FSR1_SHARD_SKIP_HALO | FSR1_SHARD_TRACE | FSR1_SHARD_DYNAMIC;

// Kinds of frame that fsr1_upscale may run on different kernels: exactly 2x (the fused / 2x-tiled kernels), any other upscale
// (the any-scale tiled kernels), and everything else (direct kernels).  Whether the EASU kernel carries the halo hand-shake
// itself is a property of the kind: RGBA16F upscales (2x and any scale) take launch_easu_h_tiled / the fused kernel, which do;
// RGBA16F downscales, FSR1_FLAG_PRECISE, fp32 and UNORM frames take kernels that do not.  The kinds are the two scale tests every
// launcher chooses by (is_2x, is_upscale, fsr1_common.cuh): a launcher that chose between kernels WITHIN a kind would have to become
// a kind of its own here, or its second kernel would be loaded lazily while flag-waiting kernels spin.
enum { kFrame2x = 0, kFrameUp = 1, kFrameOther = 2, kFrameKinds = 3 };

// One use of a slot: render size, constants, and this rank's rows for it (fsr1_shard_frame; the create-time frame otherwise).
struct FramePlan {
  uint32_t rw, rh;
  uint32_t econ[16], rcon[4];
  Rows owned, needed, window;
  Rows send[2];           // my rows the neighbour needs
  uint32_t peer_win0[2];  // first logical row of the neighbour's window
  int kind;               // kFrame*
};

// The display steps of one use of a slot (fsr1_shard_post; the create-time description otherwise): the fsr1_post minus its ops, which
// are the shard's, with copies of the caller's tile descriptors (the tiles themselves stay the caller's).
struct SlotPost {
  float lfga_amount;
  uint32_t frame;
  fsr1_image grain, dither;
  bool has_grain, has_dither;
};

}  // namespace

struct fsr1_shard {
  uint32_t in_w, in_h, out_w, out_h, format, out_format, world, rank, slots, flags;
  uint32_t post_ops;           // FSR1_POST_* of every frame (0: RGBA16F slabs in the input's format, fsr1_upscale)
  SlotPost post[kMaxSlots];    // the next use of each slot
  int device;
  // geometry of THIS rank: the output slab is fixed, the input rows are per frame
  Rows out_rows, easu_rows;
  FramePlan base;              // the create-time frame: whole resource, create sharpness (fsr1_shard_geometry)
  FramePlan plan[kMaxSlots];   // the next use of each slot
  // arena: [flags page][slot 0 window][slot 1 window]...; identical layout on every rank
  uint64_t pitch, slot_stride, arena_bytes;
  uint32_t win_rows_max;
  uint32_t min_rh;             // FSR1_SHARD_DYNAMIC: the smallest render height accepted (see the header)
  unsigned char* arena;
  unsigned char* peer[2];      // [kFromUp] = arena of rank-1, [kFromDown] = arena of rank+1 (mapped), nullptr = none
  bool peer_is_ipc[2];
  unsigned char* tmp;          // slots x rows easu_rows; null when the frames take the fused kernel (no intermediate)
  unsigned char* out;          // slots x rows out_rows, in out_format
  uint64_t out_pitch, tmp_pitch, tmp_slot_stride, out_slot_stride;
  uint32_t seq[kMaxSlots];
  cudaStream_t s_comm, s_easu, s_rcas;
  cudaEvent_t ev_in[kMaxSlots], ev_push[kMaxSlots], ev_rcas[kMaxSlots];
  bool attached;
  unsigned long long* trace;  // FSR1_SHARD_TRACE: kTraceFrames x kTraceWords globaltimer stamps (device memory), else null
  unsigned long long frames;  // frames submitted
  bool kind_ok[kFrameKinds];        // a dry frame of this kind ran at create (its kernels are loaded)
  bool inkernel_sync[kFrameKinds];  // the EASU / fused kernel of this kind of frame carries the hand-shake itself (HaloSync)
};

namespace {

Rows plan_out_rows(const fsr1_shard* s, uint32_t r) {
  return Rows{(uint32_t)((uint64_t)r * s->out_h / s->world), (uint32_t)((uint64_t)(r + 1) * s->out_h / s->world)};
}
Rows plan_easu_rows(const fsr1_shard* s, uint32_t r) {
  const Rows o = plan_out_rows(s, r);
  return fsr1::easu_rows(o.a, o.b, s->out_h);
}
// input rows of a frame `rh` rows tall
Rows plan_owned(const fsr1_shard* s, uint32_t rh, uint32_t r) {
  return Rows{(uint32_t)((uint64_t)r * rh / s->world), (uint32_t)((uint64_t)(r + 1) * rh / s->world)};
}
Rows plan_needed(const fsr1_shard* s, const uint32_t econ[16], uint32_t rh, uint32_t r) {
  const Rows e = plan_easu_rows(s, r);
  uint32_t first = 0, last = 0;
  fsr1_easu_input_rows(econ, rh, e.a, e.b, &first, &last);
  return Rows{first, last + 1};
}
Rows plan_window(const fsr1_shard* s, const uint32_t econ[16], uint32_t rh, uint32_t r) {
  const Rows o = plan_owned(s, rh, r), n = plan_needed(s, econ, rh, r);
  return Rows{o.a < n.a ? o.a : n.a, o.b > n.b ? o.b : n.b};
}

int frame_kind(const uint32_t econ[16]) {
  const float c0x = fsr1::word_as_float(econ[0]), c0y = fsr1::word_as_float(econ[1]), c0z = fsr1::word_as_float(econ[2]),
              c0w = fsr1::word_as_float(econ[3]);
  if (fsr1::is_2x(c0x, c0y, c0z, c0w)) return kFrame2x;
  return fsr1::is_upscale(c0x, c0y) ? kFrameUp : kFrameOther;
}

// The plan of frame rw x rh for this rank, with the constants context_run builds (FsrEasuCon(rw, rh, rw, rh, out_w, out_h),
// FsrRcasCon(sharpness)).  FSR1_ERR_UNSUPPORTED when some rank's halo would have to come from beyond its direct neighbours
// (true whenever a slab is taller than the halo).  *win_rows: the tallest window of any rank at this height.
int make_plan(const fsr1_shard* s, uint32_t rw, uint32_t rh, float sharpness, FramePlan* p, uint32_t* win_rows) {
  p->rw = rw;
  p->rh = rh;
  fsr1_easu_con(p->econ, (float)rw, (float)rh, (float)rw, (float)rh, (float)s->out_w, (float)s->out_h);
  fsr1_rcas_con(p->rcon, sharpness);
  p->kind = frame_kind(p->econ);
  uint32_t wmax = 0;
  for (uint32_t r = 0; r < s->world; r++) {
    const Rows n = plan_needed(s, p->econ, rh, r), w = plan_window(s, p->econ, rh, r);
    const uint32_t lo = r == 0 ? 0 : plan_owned(s, rh, r - 1).a, hi = r + 1 == s->world ? rh : plan_owned(s, rh, r + 1).b;
    if (n.a < lo || n.b > hi) return FSR1_ERR_UNSUPPORTED;
    if (w.b - w.a > wmax) wmax = w.b - w.a;
  }
  if (win_rows) *win_rows = wmax;
  const uint32_t rank = s->rank;
  p->owned = plan_owned(s, rh, rank);
  p->needed = plan_needed(s, p->econ, rh, rank);
  p->window = plan_window(s, p->econ, rh, rank);
  for (int side = 0; side < 2; side++) {
    p->send[side] = Rows{0, 0};
    p->peer_win0[side] = 0;
    const bool has = side == kFromUp ? rank > 0 : rank + 1 < s->world;
    if (!has) continue;
    const uint32_t peer = side == kFromUp ? rank - 1 : rank + 1;
    const Rows pn = plan_needed(s, p->econ, rh, peer);
    const uint32_t a = p->owned.a > pn.a ? p->owned.a : pn.a, b = p->owned.b < pn.b ? p->owned.b : pn.b;
    if (b > a) p->send[side] = Rows{a, b};
    p->peer_win0[side] = plan_window(s, p->econ, rh, peer).a;
  }
  return FSR1_OK;
}

// FSR1_SHARD_DYNAMIC: marks, per rank, the offsets into its window of the rows its push to each side reads and the rows the
// neighbour on each side writes, for frames of height rh; false when a row the lower neighbour writes is one the push UP reads,
// or a row the upper neighbour writes is one the push DOWN reads, for this or for a height marked before (see the header).
bool mark_push_rows(const fsr1_shard* s, const uint32_t econ[16], uint32_t rh, std::vector<std::vector<uint8_t>>& marks) {
  enum : uint8_t { kReadUp = 1, kReadDown = 2, kWriteFromUp = 4, kWriteFromDown = 8 };
  for (uint32_t r = 0; r < s->world; r++) {
    const Rows o = plan_owned(s, rh, r), n = plan_needed(s, econ, rh, r), w = plan_window(s, econ, rh, r);
    std::vector<uint8_t>& m = marks[r];
    if (m.size() < w.b - w.a) m.resize(w.b - w.a, 0);
    auto mark = [&](uint32_t a, uint32_t b, uint8_t bit, uint8_t other) {  // rows [a, b)
      for (uint32_t y = a; y < b; y++) {
        if (m[y - w.a] & other) return false;
        m[y - w.a] |= bit;
      }
      return true;
    };
    for (int side = 0; side < 2; side++) {
      const bool has = side == kFromUp ? r > 0 : r + 1 < s->world;
      if (!has) continue;
      const uint32_t peer = side == kFromUp ? r - 1 : r + 1;
      const Rows po = plan_owned(s, rh, peer), pn = plan_needed(s, econ, rh, peer);
      const uint32_t sa = o.a > pn.a ? o.a : pn.a, sb = o.b < pn.b ? o.b : pn.b;  // my rows the neighbour needs
      const uint32_t ra = po.a > n.a ? po.a : n.a, rb = po.b < n.b ? po.b : n.b;  // the neighbour's rows I need
      const bool ok = side == kFromUp ? mark(sa, sb, kReadUp, kWriteFromDown) && mark(ra, rb, kWriteFromUp, kReadDown)
                                      : mark(sa, sb, kReadDown, kWriteFromUp) && mark(ra, rb, kWriteFromDown, kReadUp);
      if (!ok) return false;
    }
  }
  return true;
}

int cuda_rc(cudaError_t e) { return e == cudaSuccess ? FSR1_OK : FSR1_ERR_CUDA; }

struct DeviceGuard {  // calls may come from a thread whose current device is another GPU (one process, several ranks)
  int prev;
  explicit DeviceGuard(int dev) : prev(-1) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

fsr1_image make_img(void* data, uint64_t pitch, uint32_t w, uint32_t h, uint32_t row0, uint32_t rows, uint32_t fmt) {
  fsr1_image im;
  im.data = data; im.pitch_bytes = pitch; im.width = w; im.height = h; im.row0 = row0; im.rows = rows; im.format = fmt; im.reserved = 0;
  return im;
}
unsigned char* window_of(const fsr1_shard* s, unsigned char* arena, uint32_t slot) { return arena + kFlagBytes + (uint64_t)slot * s->slot_stride; }
fsr1_image tmp_of(const fsr1_shard* s, uint32_t slot) {
  return make_img(s->tmp + (uint64_t)slot * s->tmp_slot_stride, s->tmp_pitch, s->out_w, s->out_h, s->easu_rows.a,
                  s->easu_rows.b - s->easu_rows.a, easu_out_format(s->format));
}
uint32_t kernel_flags(const fsr1_shard* s) { return (s->flags & ~kShardFlags) | FSR1_FLAG_FUSED; }

void set_slot_post(fsr1_shard* s, uint32_t slot, const fsr1_post* post) {
  SlotPost& d = s->post[slot];
  d.lfga_amount = post->lfga_amount;
  d.frame = post->frame;
  d.has_grain = (s->post_ops & FSR1_POST_LFGA) && post->grain;
  d.has_dither = (s->post_ops & (FSR1_POST_TEPD8 | FSR1_POST_TEPD10)) && post->dither;
  if (d.has_grain) d.grain = *post->grain;
  if (d.has_dither) d.dither = *post->dither;
}

// The frame described by slot `slot` (its plan and post) on stream `st`: fsr1_upscale_post, which is fsr1_upscale without post ops,
// with the neighbour hand-shake `sync` (fsr1::upscale_post).
int launch_frame(fsr1_shard* s, uint32_t slot, cudaStream_t st, const fsr1::HaloSync* sync, bool* sync_taken) {
  const FramePlan& p = s->plan[slot];
  fsr1_image win, out, tmp;
  fsr1_shard_window(s, slot, &win);
  fsr1_shard_output(s, slot, &out);
  if (s->tmp) tmp = tmp_of(s, slot);
  const SlotPost& d = s->post[slot];
  const fsr1_post post = {s->post_ops, d.lfga_amount, d.has_grain ? &d.grain : nullptr, d.has_dither ? &d.dither : nullptr, d.frame, 0};
  return fsr1::upscale_post(&win, s->tmp ? &tmp : nullptr, &out, p.econ, p.rcon, s->post_ops ? &post : nullptr, s->out_rows.a,
                            s->out_rows.b, kernel_flags(s), st, sync, sync_taken);
}

// One dry frame `p` on the zero-filled slot 0 (no halo protocol), through the intermediate if there is one: loads the kernels
// such a frame takes and tells whether they carry the halo hand-shake.  Leaves slot 0 described as `p`.
int dry_frame(fsr1_shard* s, const FramePlan& p, bool* inkernel) {
  s->plan[0] = p;
  const fsr1::HaloSync none = {};
  *inkernel = false;
  return launch_frame(s, 0, s->s_easu, &none, inkernel);
}

}  // namespace

extern "C" {

int fsr1_shard_create(fsr1_shard** out_sh, uint32_t in_w, uint32_t in_h, uint32_t out_w, uint32_t out_h, uint32_t format,
                      uint32_t world, uint32_t rank, uint32_t slots, float sharpness_stops, uint32_t flags) {
  return fsr1_shard_create_post(out_sh, in_w, in_h, out_w, out_h, format, easu_out_format(format), nullptr, world, rank, slots, sharpness_stops,
                                flags);
}

int fsr1_shard_create_post(fsr1_shard** out_sh, uint32_t in_w, uint32_t in_h, uint32_t out_w, uint32_t out_h, uint32_t format,
                           uint32_t out_format, const fsr1_post* post, uint32_t world, uint32_t rank, uint32_t slots, float sharpness_stops,
                           uint32_t flags) {
  if (!out_sh || !in_w || !in_h || !out_w || !out_h || !world || rank >= world || !slots || slots > kMaxSlots) return FSR1_ERR_INVALID_ARGUMENT;
  const int bpp = bytes_per_pixel(format), out_bpp = bytes_per_pixel(out_format);
  if (!bpp || !out_bpp) return FSR1_ERR_INVALID_ARGUMENT;
  if (world > in_h || world > out_h) return FSR1_ERR_INVALID_ARGUMENT;  // no empty slabs
  // the windows are linear memory the ranks export to each other, and the slabs the shard's own
  if (flags & (FSR1_FLAG_IN_SURFACE | FSR1_FLAG_OUT_SURFACE | FSR1_FLAG_IN_TEXTURE)) return FSR1_ERR_UNSUPPORTED;
  // the display steps: fsr1_upscale_post's rules, before any CUDA call; without them the slabs are in the input's format
  const uint32_t post_ops = post ? post->ops : 0u;
  if (post_ops) {
    const int rc = fsr1::post_rules(post, format, out_format, flags & ~kShardFlags);
    if (rc != FSR1_OK) return rc;
  } else if (out_format != easu_out_format(format)) {
    return FSR1_ERR_UNSUPPORTED;
  }
  fsr1_shard* s = new (std::nothrow) fsr1_shard();
  if (!s) return FSR1_ERR_INVALID_ARGUMENT;
  memset(s, 0, sizeof *s);
  s->in_w = in_w; s->in_h = in_h; s->out_w = out_w; s->out_h = out_h; s->format = format; s->out_format = out_format;
  s->world = world; s->rank = rank; s->slots = slots; s->flags = flags;
  s->post_ops = post_ops;
  if (post_ops)
    for (uint32_t i = 0; i < slots; i++) set_slot_post(s, i, post);
  if (cudaGetDevice(&s->device) != cudaSuccess) { delete s; return FSR1_ERR_NO_DEVICE; }
  const bool dynamic = (flags & FSR1_SHARD_DYNAMIC) != 0;
  s->out_rows = plan_out_rows(s, rank);
  s->easu_rows = plan_easu_rows(s, rank);
  // every rank's halo must come from its direct neighbours only (true whenever a slab is taller than the halo)
  if (make_plan(s, in_w, in_h, sharpness_stops, &s->base, &s->win_rows_max) != FSR1_OK) { delete s; return FSR1_ERR_UNSUPPORTED; }
  // FSR1_SHARD_DYNAMIC: the render heights accepted are those from in_h down to the first height whose push rows would meet another
  // accepted height's (mark_push_rows) that pass the same rule; the windows take the tallest of them.  All of it is a function of
  // the shard's arguments only: the same on every rank.  The same scan finds one render size of each kind of frame for the dry
  // frames below (the create-time frame first, for its own kind).
  uint32_t rep_w[kFrameKinds] = {0, 0, 0}, rep_h[kFrameKinds] = {0, 0, 0};
  s->min_rh = in_h;
  if (dynamic) {
    const uint32_t fit_w = in_w < out_w ? in_w : out_w;
    const uint32_t cand_w[4] = {in_w, fit_w, fit_w - 1, out_w / 2};  // fit_w - 1, out_w / 2 may be 0: skipped
    std::vector<std::vector<uint8_t>> marks(world);
    for (uint32_t rh = in_h; rh >= world; rh--) {
      FramePlan p;
      uint32_t win_rows = 0;
      if (make_plan(s, in_w, rh, sharpness_stops, &p, &win_rows) != FSR1_OK) continue;  // the rule depends on rh only
      if (!mark_push_rows(s, p.econ, rh, marks)) break;
      s->min_rh = rh;
      if (win_rows > s->win_rows_max) s->win_rows_max = win_rows;
      for (uint32_t rw : cand_w) {
        if (rw == 0 || rw > in_w) continue;
        uint32_t econ[16];
        fsr1_easu_con(econ, (float)rw, (float)rh, (float)rw, (float)rh, (float)out_w, (float)out_h);
        const int k = frame_kind(econ);
        if (!rep_h[k]) { rep_w[k] = rw; rep_h[k] = rh; }
      }
    }
  }
  for (uint32_t i = 0; i < slots; i++) s->plan[i] = s->base;
  s->pitch = ((uint64_t)in_w * bpp + 127) & ~(uint64_t)127;
  s->slot_stride = ((uint64_t)s->win_rows_max * s->pitch + 255) & ~(uint64_t)255;
  s->arena_bytes = kFlagBytes + s->slot_stride * slots;
  s->out_pitch = ((uint64_t)out_w * out_bpp + 127) & ~(uint64_t)127;
  s->tmp_pitch = ((uint64_t)out_w * bytes_per_pixel(easu_out_format(format)) + 127) & ~(uint64_t)127;  // the intermediate: EASU's output format
  s->tmp_slot_stride = (uint64_t)(s->easu_rows.b - s->easu_rows.a) * s->tmp_pitch;
  s->out_slot_stride = (uint64_t)(s->out_rows.b - s->out_rows.a) * s->out_pitch;
  cudaError_t e;
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // numerically lowest = most urgent
  // cudaMalloc (not a pool / VMM allocation): the arena must be exportable through cudaIpcGetMemHandle
  if ((e = cudaMalloc((void**)&s->arena, s->arena_bytes)) != cudaSuccess || (e = cudaMemset(s->arena, 0, s->arena_bytes)) != cudaSuccess ||
      (e = cudaMalloc((void**)&s->out, s->out_slot_stride * slots)) != cudaSuccess ||
      (e = cudaStreamCreateWithPriority(&s->s_comm, cudaStreamNonBlocking, prio_hi)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&s->s_easu, cudaStreamNonBlocking)) != cudaSuccess ||
      (e = cudaStreamCreateWithFlags(&s->s_rcas, cudaStreamNonBlocking)) != cudaSuccess) {
    fsr1_shard_destroy(s);
    return FSR1_ERR_CUDA;
  }
  if ((flags & FSR1_SHARD_TRACE) && (cudaMalloc((void**)&s->trace, sizeof(unsigned long long) * kTraceFrames * kTraceWords) != cudaSuccess ||
                                     cudaMemset(s->trace, 0, sizeof(unsigned long long) * kTraceFrames * kTraceWords) != cudaSuccess)) {
    fsr1_shard_destroy(s);
    return FSR1_ERR_CUDA;
  }
  for (uint32_t i = 0; i < slots; i++) {
    if (cudaEventCreateWithFlags(&s->ev_in[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s->ev_push[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s->ev_rcas[i], cudaEventDisableTiming) != cudaSuccess) {
      fsr1_shard_destroy(s);
      return FSR1_ERR_CUDA;
    }
  }
  if (world > 1) {
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, halo_push_kernel) != cudaSuccess || cudaFuncGetAttributes(&fa, halo_wait_kernel) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, credit_signal_kernel) != cudaSuccess) {
      fsr1_shard_destroy(s);
      return FSR1_ERR_CUDA;
    }
  }
  // One dry frame on the zero-filled slot 0 (no halo protocol).  Every frame of a static shard has this frame's format, scale, layout
  // and options, so it decides for all of them:
  //  - whether they take the fused EASU->RCAS kernel.  It is tried first, without an intermediate; only a configuration it does not
  //    cover (fsr1_upscale then needs `tmp`) gets the intermediate, 66 MB per slot at 1080p->4K RGBA16F, and runs the frame again
  //    through the two kernels;
  //  - whether the kernel takes the halo hand-shake itself (null pointers: a no-op inside the kernel);
  //  - and it loads every kernel a frame uses NOW.  CUDA loads kernels lazily, on first launch, and loading may synchronise the
  //    context: a first-use load issued while a flag-waiting kernel spins would wait for that kernel, which (several ranks in ONE
  //    process) may be waiting for work this very host thread has not submitted yet.
  // A dynamic shard's frames differ in scale, so it allocates the intermediate up front (any frame that is not exactly 2x needs it;
  // its size depends on the fixed output slab only) and runs one dry frame of every kind a frame can be: the create-time frame for
  // its kind, a representative render size for each other kind.  A kind whose dry frame is refused with FSR1_ERR_UNSUPPORTED (the
  // flags exclude it) is refused by fsr1_shard_frame as well.
  // With display steps every frame is fsr1_upscale_post with the shard's ops and output format, so the dry frames run it with the
  // create-time description and load the post kernels (the fused post kernel, or tiled EASU + the RCAS post kernel; the srtm_in
  // variants with FSR1_FLAG_SRTM_INPUT): which of them a frame takes depends on its kind, the flags and the output format only.
  bool inkernel = false;
  if (!dynamic) {
    int rc = dry_frame(s, s->base, &inkernel);
    if (rc != FSR1_OK) {
      if ((e = cudaMalloc((void**)&s->tmp, s->tmp_slot_stride * slots)) != cudaSuccess) { fsr1_shard_destroy(s); return FSR1_ERR_CUDA; }
      rc = dry_frame(s, s->base, &inkernel);
    }
    if (rc != FSR1_OK) { fsr1_shard_destroy(s); return rc; }
    s->kind_ok[s->base.kind] = true;
    s->inkernel_sync[s->base.kind] = inkernel;
  } else {
    if ((e = cudaMalloc((void**)&s->tmp, s->tmp_slot_stride * slots)) != cudaSuccess) { fsr1_shard_destroy(s); return FSR1_ERR_CUDA; }
    for (int k = 0; k < kFrameKinds; k++) {
      if (!rep_h[k]) continue;
      FramePlan p;
      if (k == s->base.kind) p = s->base;
      else make_plan(s, rep_w[k], rep_h[k], sharpness_stops, &p, nullptr);  // passed the rule in the scan
      const int rc = dry_frame(s, p, &inkernel);
      if (rc == FSR1_ERR_UNSUPPORTED && k != s->base.kind) continue;
      if (rc != FSR1_OK) { fsr1_shard_destroy(s); return rc; }
      s->kind_ok[k] = true;
      s->inkernel_sync[k] = inkernel;
    }
  }
  s->plan[0] = s->base;
  if ((e = cudaDeviceSynchronize()) != cudaSuccess) { fsr1_shard_destroy(s); return FSR1_ERR_CUDA; }  // flags are zero before anyone attaches
  s->attached = world == 1 || (flags & FSR1_SHARD_SKIP_HALO);
  *out_sh = s;
  return FSR1_OK;
}

void fsr1_shard_destroy(fsr1_shard* s) {
  if (!s) return;
  DeviceGuard g(s->device);
  cudaDeviceSynchronize();
  for (int side = 0; side < 2; side++)
    if (s->peer[side] && s->peer_is_ipc[side]) cudaIpcCloseMemHandle(s->peer[side]);
  for (uint32_t i = 0; i < s->slots && i < kMaxSlots; i++) {
    if (s->ev_in[i]) cudaEventDestroy(s->ev_in[i]);
    if (s->ev_push[i]) cudaEventDestroy(s->ev_push[i]);
    if (s->ev_rcas[i]) cudaEventDestroy(s->ev_rcas[i]);
  }
  if (s->s_comm) cudaStreamDestroy(s->s_comm);
  if (s->s_easu) cudaStreamDestroy(s->s_easu);
  if (s->s_rcas) cudaStreamDestroy(s->s_rcas);
  cudaFree(s->arena);
  cudaFree(s->trace);
  cudaFree(s->tmp);
  cudaFree(s->out);
  delete s;
}

int fsr1_shard_geometry(const fsr1_shard* s, fsr1_shard_info* info) {
  if (!s || !info) return FSR1_ERR_INVALID_ARGUMENT;
  info->out_row0 = s->out_rows.a; info->out_row1 = s->out_rows.b;
  info->easu_row0 = s->easu_rows.a; info->easu_row1 = s->easu_rows.b;
  const FramePlan& p = s->base;
  info->owned_row0 = p.owned.a; info->owned_row1 = p.owned.b;
  info->needed_row0 = p.needed.a; info->needed_row1 = p.needed.b;
  info->window_row0 = p.window.a; info->window_row1 = p.window.b;
  info->send_up_row0 = p.send[kFromUp].a; info->send_up_row1 = p.send[kFromUp].b;
  info->send_down_row0 = p.send[kFromDown].a; info->send_down_row1 = p.send[kFromDown].b;
  info->halo_recv_bytes = (uint64_t)((p.owned.a - p.window.a) + (p.window.b - p.owned.b)) * s->in_w * bytes_per_pixel(s->format);
  info->arena_bytes = s->arena_bytes;
  return FSR1_OK;
}

int fsr1_shard_export(const fsr1_shard* s, void* handle) {
  if (!s || !handle) return FSR1_ERR_INVALID_ARGUMENT;
  static_assert(sizeof(cudaIpcMemHandle_t) == FSR1_SHARD_HANDLE_BYTES, "handle size");
  DeviceGuard g(s->device);
  cudaIpcMemHandle_t h;
  if (cudaIpcGetMemHandle(&h, s->arena) != cudaSuccess) return FSR1_ERR_CUDA;
  memcpy(handle, &h, sizeof h);
  return FSR1_OK;
}

void* fsr1_shard_arena(const fsr1_shard* s) { return s ? s->arena : nullptr; }

static int attach_done(fsr1_shard* s) {
  s->attached = (s->rank == 0 || s->peer[kFromUp]) && (s->rank + 1 == s->world || s->peer[kFromDown]);
  return s->attached ? FSR1_OK : FSR1_ERR_INVALID_ARGUMENT;
}

int fsr1_shard_attach(fsr1_shard* s, const void* handles, uint32_t count) {
  if (!s || !handles || count != s->world) return FSR1_ERR_INVALID_ARGUMENT;
  DeviceGuard g(s->device);
  for (int side = 0; side < 2; side++) {
    const bool has = side == kFromUp ? s->rank > 0 : s->rank + 1 < s->world;
    if (!has || s->peer[side]) continue;
    const uint32_t peer = side == kFromUp ? s->rank - 1 : s->rank + 1;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const unsigned char*)handles + (size_t)peer * FSR1_SHARD_HANDLE_BYTES, sizeof h);
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) return FSR1_ERR_CUDA;
    s->peer[side] = (unsigned char*)p;
    s->peer_is_ipc[side] = true;
  }
  return attach_done(s);
}

int fsr1_shard_attach_local(fsr1_shard* s, fsr1_shard* up, fsr1_shard* down) {
  if (!s) return FSR1_ERR_INVALID_ARGUMENT;
  DeviceGuard g(s->device);
  fsr1_shard* nb[2] = {up, down};
  for (int side = 0; side < 2; side++) {
    const bool has = side == kFromUp ? s->rank > 0 : s->rank + 1 < s->world;
    if (!has) continue;
    fsr1_shard* n = nb[side];
    if (!n || n->world != s->world || n->rank != (side == kFromUp ? s->rank - 1 : s->rank + 1) || n->arena_bytes != s->arena_bytes)
      return FSR1_ERR_INVALID_ARGUMENT;
    if (n->device != s->device) {
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, s->device, n->device) != cudaSuccess || !can) return FSR1_ERR_UNSUPPORTED;
      cudaError_t e = cudaDeviceEnablePeerAccess(n->device, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) return FSR1_ERR_CUDA;
    }
    s->peer[side] = n->arena;
    s->peer_is_ipc[side] = false;
  }
  return attach_done(s);
}

int fsr1_shard_frame(fsr1_shard* s, uint32_t slot, uint32_t render_w, uint32_t render_h, float sharpness_stops) {
  if (!s || !(s->flags & FSR1_SHARD_DYNAMIC) || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  if (!render_w || !render_h || render_w > s->in_w || render_h > s->in_h || s->world > render_h) return FSR1_ERR_INVALID_ARGUMENT;
  if (render_h < s->min_rh) return FSR1_ERR_UNSUPPORTED;  // a neighbour's halo rows could meet rows my push of another height reads
  FramePlan p;
  uint32_t win_rows = 0;
  const int rc = make_plan(s, render_w, render_h, sharpness_stops, &p, &win_rows);
  if (rc != FSR1_OK) return rc;
  // a kind of frame whose dry frame the kernels refused at create (its kernels are not loaded), and a window beyond the capacity
  // (cannot happen: create sized the windows over every accepted height)
  if (!s->kind_ok[p.kind] || win_rows > s->win_rows_max) return FSR1_ERR_UNSUPPORTED;
  s->plan[slot] = p;
  return FSR1_OK;
}

int fsr1_shard_input(const fsr1_shard* s, uint32_t slot, fsr1_image* owned) {
  if (!s || !owned || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  const FramePlan& p = s->plan[slot];
  *owned = make_img(window_of(s, s->arena, slot) + (uint64_t)(p.owned.a - p.window.a) * s->pitch, s->pitch, p.rw, p.rh, p.owned.a,
                    p.owned.b - p.owned.a, s->format);
  return FSR1_OK;
}

int fsr1_shard_window(const fsr1_shard* s, uint32_t slot, fsr1_image* window) {
  if (!s || !window || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  const FramePlan& p = s->plan[slot];
  *window = make_img(window_of(s, s->arena, slot), s->pitch, p.rw, p.rh, p.window.a, p.window.b - p.window.a, s->format);
  return FSR1_OK;
}

int fsr1_shard_output(const fsr1_shard* s, uint32_t slot, fsr1_image* out) {
  if (!s || !out || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  *out = make_img(s->out + (uint64_t)slot * s->out_slot_stride, s->out_pitch, s->out_w, s->out_h, s->out_rows.a, s->out_rows.b - s->out_rows.a,
                  s->out_format);
  return FSR1_OK;
}

int fsr1_shard_post(fsr1_shard* s, uint32_t slot, const fsr1_post* post) {
  if (!s || slot >= s->slots || !post || !s->post_ops || post->ops != s->post_ops) return FSR1_ERR_INVALID_ARGUMENT;
  const int rc = fsr1::post_rules(post, s->format, s->out_format, s->flags & ~kShardFlags);
  if (rc != FSR1_OK) return rc;
  set_slot_post(s, slot, post);
  return FSR1_OK;
}

int fsr1_shard_submit(fsr1_shard* s, uint32_t slot, void* stream) {
  if (!s || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  if (!s->attached) return FSR1_ERR_INVALID_ARGUMENT;
  DeviceGuard g(s->device);
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  const bool one_stream = (s->flags & FSR1_SHARD_ONE_STREAM) != 0;
  cudaStream_t se = s->s_easu, sr = one_stream ? s->s_easu : s->s_rcas;
  const uint32_t q = ++s->seq[slot];
  struct FrameCount { fsr1_shard* s; ~FrameCount() { s->frames++; } } frame_count{s};
  uint32_t* flags = reinterpret_cast<uint32_t*>(s->arena);
  cudaError_t e;
  if ((e = cudaEventRecord(s->ev_in[slot], caller)) != cudaSuccess) return cuda_rc(e);
  const bool skip_halo = (s->flags & FSR1_SHARD_SKIP_HALO) != 0;  // measurement only: what the frame costs without the exchange
  const bool up = s->rank > 0 && !skip_halo, down = s->rank + 1 < s->world && !skip_halo;
  const FramePlan& p = s->plan[slot];  // this use of the slot: both ends of a push compute the same rows from it
  if (up || down) {
    PushSide ps[2];
    for (int side = 0; side < 2; side++) {
      ps[side] = PushSide{nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr};
      const bool has = side == kFromUp ? up : down;
      if (!has) continue;
      const Rows r = p.send[side];
      uint32_t* pf = reinterpret_cast<uint32_t*>(s->peer[side]);
      ps[side].src = reinterpret_cast<const uint4*>(window_of(s, s->arena, slot) + (uint64_t)(r.a - p.window.a) * s->pitch);
      ps[side].dst = reinterpret_cast<uint4*>(window_of(s, s->peer[side], slot) + (uint64_t)(r.a - p.peer_win0[side]) * s->pitch);
      ps[side].n16 = (uint32_t)((uint64_t)(r.b - r.a) * s->pitch / 16);
      ps[side].credit = flags + credit_idx(slot, side);
      ps[side].parts_done = flags + push_cnt_idx(slot, side);
      ps[side].trace = s->trace ? s->trace + (size_t)(s->frames % kTraceFrames) * kTraceWords : nullptr;
      // I am the neighbour's lower (upper) peer when I push up (down)
      ps[side].ready = pf + ready_idx(slot, side == kFromUp ? kFromDown : kFromUp);
    }
    if ((e = cudaStreamWaitEvent(s->s_comm, s->ev_in[slot], 0)) != cudaSuccess) return cuda_rc(e);
    halo_push_kernel<<<2 * kPushParts, 32, 0, s->s_comm>>>(ps[kFromUp], ps[kFromDown], q, flags + kStatusIdx);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_rc(e);
    if ((e = cudaEventRecord(s->ev_push[slot], s->s_comm)) != cudaSuccess) return cuda_rc(e);
  }
  // fused whenever the kernel covers the frame (a static shard allocated no intermediate then), else EASU + RCAS through `tmp`
  // The whole frame runs on ONE stream, consecutive frames on the two streams in turn: the tail of frame i overlaps the start of
  // frame i+1 (and with two kernels, RCAS of frame i (ALU / XU / HBM-bound) overlaps EASU of frame i+1 (FMA-pipe-bound)) without an
  // event between the kernels of a frame.
  cudaStream_t sk = (!one_stream && (s->frames & 1)) ? sr : se;
  if ((e = cudaStreamWaitEvent(sk, s->ev_in[slot], 0)) != cudaSuccess) return cuda_rc(e);
  if (q > 1 && !one_stream && (e = cudaStreamWaitEvent(sk, s->ev_rcas[slot], 0)) != cudaSuccess) return cuda_rc(e);  // the slot's intermediate / output are free
  fsr1::HaloSync hs = {};
  hs.ready[kFromUp] = up ? flags + ready_idx(slot, kFromUp) : nullptr;
  hs.ready[kFromDown] = down ? flags + ready_idx(slot, kFromDown) : nullptr;
  hs.credit[kFromUp] = up ? reinterpret_cast<uint32_t*>(s->peer[kFromUp]) + credit_idx(slot, kFromDown) : nullptr;
  hs.credit[kFromDown] = down ? reinterpret_cast<uint32_t*>(s->peer[kFromDown]) + credit_idx(slot, kFromUp) : nullptr;
  hs.counter = flags + counter_idx(slot);
  hs.status = flags + kStatusIdx;
  hs.trace = s->trace ? s->trace + (size_t)(s->frames % kTraceFrames) * kTraceWords : nullptr;
  hs.seq = q;
  const bool shake = up || down, inkernel = shake && s->inkernel_sync[p.kind];
  if (shake && !inkernel) {
    halo_wait_kernel<<<1, 32, 0, sk>>>(hs.ready[kFromUp], hs.ready[kFromDown], q, flags + kStatusIdx);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_rc(e);
  }
  bool took = false;
  const int rc = launch_frame(s, slot, sk, inkernel ? &hs : nullptr, &took);
  if (rc != FSR1_OK) return rc;
  if (inkernel && !took) return FSR1_ERR_UNSUPPORTED;  // cannot happen: the capability was probed with this configuration
  if (shake && !inkernel) {
    credit_signal_kernel<<<1, 32, 0, sk>>>(hs.credit[kFromUp], hs.credit[kFromDown], q);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_rc(e);
  }
  if ((e = cudaEventRecord(s->ev_rcas[slot], sk)) != cudaSuccess) return cuda_rc(e);
  return FSR1_OK;
}

int fsr1_shard_wait(fsr1_shard* s, uint32_t slot, void* stream) {
  if (!s || slot >= s->slots) return FSR1_ERR_INVALID_ARGUMENT;
  if (s->seq[slot] == 0) return FSR1_OK;
  DeviceGuard g(s->device);
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if ((e = cudaStreamWaitEvent(caller, s->ev_rcas[slot], 0)) != cudaSuccess) return cuda_rc(e);
  if (s->world > 1 && !(s->flags & FSR1_SHARD_SKIP_HALO) && (e = cudaStreamWaitEvent(caller, s->ev_push[slot], 0)) != cudaSuccess)
    return cuda_rc(e);  // my rows have left
  return FSR1_OK;
}

int fsr1_shard_trace(fsr1_shard* s, uint64_t* out, uint32_t max_frames, uint32_t* n_frames) {
  if (!s || !out || !n_frames) return FSR1_ERR_INVALID_ARGUMENT;
  *n_frames = 0;
  if (!s->trace) return FSR1_OK;
  DeviceGuard g(s->device);
  uint32_t n = (uint32_t)(s->frames < kTraceFrames ? s->frames : kTraceFrames);
  if (n > max_frames) n = max_frames;
  // oldest first: frames [frames - n, frames)
  for (uint32_t i = 0; i < n; i++) {
    const unsigned long long f = s->frames - n + i;
    if (cudaMemcpy(out + (size_t)i * kTraceWords, s->trace + (size_t)(f % kTraceFrames) * kTraceWords, sizeof(unsigned long long) * kTraceWords,
                   cudaMemcpyDeviceToHost) != cudaSuccess)
      return FSR1_ERR_CUDA;
  }
  *n_frames = n;
  return FSR1_OK;
}

int fsr1_shard_status(fsr1_shard* s) {
  if (!s) return FSR1_ERR_INVALID_ARGUMENT;
  DeviceGuard g(s->device);
  uint32_t st = 0;
  if (cudaMemcpy(&st, reinterpret_cast<uint32_t*>(s->arena) + kStatusIdx, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return FSR1_ERR_CUDA;
  if (st != 0) fsr1::set_last_detail(1000 + (int)st + 10 * (int)s->rank);  // 1 / 2: push up / down starved of credit; 3 / 4: halo from above / below never came
  return st == 0 ? FSR1_OK : FSR1_ERR_TIMEOUT;
}

}  // extern "C"
