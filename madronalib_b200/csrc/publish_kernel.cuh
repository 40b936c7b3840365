// publish_kernel.cuh -- K14: published signals of G instruments, the reference's SignalProcessor::PublishedSignal
// (source/app/MLSignalProcessor.h:28-105, MLSignalProcessor.cpp:11-38, the ring of source/DSP/MLDSPBuffer.h:47-384).
//
// Per instrument and signal the reference keeps a ring of `size` floats (2^bitsToContain(maxFrames * channels *
// maxVoices), at least 64), a write and a read index in [0, 2 size) and one decimation counter c shared by every
// voice.  Within a vector the stores arrive in voice order, then in call order within processVoice; that sequence
// carries across vectors and calls.  A store of n frames writes frame f exactly when (c + f + 1) % 2^octavesDown == 0,
// so over a chunk of T vectors the k-th frame of the whole sequence is written iff (c + k + 1) is a multiple of
// 2^octavesDown: the q-th written frame is frame k_q = (q + 1) 2^octavesDown - c - 1, and the chunk writes
// W = ((c + total) >> octavesDown) * channels floats and leaves c' = (c + total) & (2^octavesDown - 1).
//
// No single write exceeds the ring (frames <= maxFrames is checked where the bank is made), so the reference's
// clobbering writes compose: after the chunk, readable = min(readable + W, size), the write index moves by W, and
// of the W floats only the last min(W, size) survive.  Each of those goes to its own slot, so the lanes of one warp
// place them in parallel: one warp per (signal, instrument), no atomics, no synchronisation beyond the warp.
#pragma once
#include "ops.cuh"

namespace mlb
{
constexpr int kPubWarps = 8;          // (signal, instrument) items per 256-thread CTA
constexpr int kPubMaxSignals = 16;    // MLB_PUBLISHED_MAX_SIGNALS
constexpr int kPubMaxStores = 64;     // MLB_PUBLISHED_MAX_STORES

struct PubSignal
{
  int channels, octaves, size;  // size: ring floats, a power of two
  int first_item, n_items;      // its stores: items [first_item, first_item + n_items) in call order
  int frames;                   // sum of its stores' frames: frames per voice and vector
  long long ring;               // offset of instrument 0's ring in PubArgs::ring; instrument g at ring + g * size
};

struct PubItem
{
  int frames, plane;  // plane: first of the store's `channels` rows, counted from the first published plane
};

struct PubArgs
{
  const float* rows;      // [T][stride][V][64]: published planes at [plane0, plane0 + n_pub)
  float* ring;            // every ring, PubSignal::ring
  uint32_t* state;        // [n_signals][G][3]: write index, read index, counter
  const int32_t* first;   // [G] first voice of instrument g
  const int32_t* count;   // [G] its voices
  int V, G, T, stride, plane0, n_signals;
  PubSignal sig[kPubMaxSignals];
  PubItem item[kPubMaxStores];
};

__global__ void __launch_bounds__(32 * kPubWarps) publish_kernel(const PubArgs a)
{
  const int w = blockIdx.x * kPubWarps + (threadIdx.x >> 5);
  if (w >= a.n_signals * a.G) return;
  const int lane = threadIdx.x & 31;
  const int s = w / a.G, g = w - s * a.G;
  const PubSignal& sg = a.sig[s];
  uint32_t* st = a.state + (size_t)w * 3;
  const uint32_t w0 = st[0], r0 = st[1], c0 = st[2];
  const uint32_t size = (uint32_t)sg.size, dist = 2 * size - 1;
  const long long perVector = (long long)__ldg(a.count + g) * sg.frames;  // frames of one vector, all voices
  const long long total = perVector * a.T;
  const long long written = (((long long)c0 + total) >> sg.octaves) * sg.channels;  // floats this chunk writes
  if (written > 0)
  {
    const int lane0 = __ldg(a.first + g);
    float* ring = a.ring + sg.ring + (long long)g * sg.size;
    for (long long j = written > size ? written - size : 0; j < written; j += 32)
    {
      const long long jj = j + lane;
      if (jj >= written) break;
      const long long q = jj / sg.channels;
      const int ch = (int)(jj - q * sg.channels);
      const long long k = ((q + 1) << sg.octaves) - (long long)c0 - 1;  // frame of the chunk's store sequence
      const long long t = k / perVector;
      const long long rem = k - t * perVector;
      const int v = (int)(rem / sg.frames);
      int f = (int)(rem - (long long)v * sg.frames);
      int it = sg.first_item;
      while (f >= a.item[it].frames) f -= a.item[it].frames, ++it;
      const float x = a.rows[(((size_t)t * a.stride + a.plane0 + a.item[it].plane + ch) * a.V + lane0 + v) * MLB_BLOCK + f];
      ring[((size_t)w0 + (size_t)jj) & (size - 1)] = x;
    }
  }
  __syncwarp();
  if (lane == 0)
  {
    const uint32_t avail = (w0 - r0) & dist;
    const long long a2 = (long long)avail + written;
    const uint32_t nw = (uint32_t)((w0 + (unsigned long long)written) & dist);
    st[0] = nw;
    st[1] = (nw - (uint32_t)(a2 < size ? a2 : size)) & dist;
    st[2] = (uint32_t)(((long long)c0 + total) & ((1ll << sg.octaves) - 1));
  }
}

// The batched reads of one signal, one warp per instrument (MLSignalProcessor.cpp:19-38, MLDSPBuffer.h:199-218,
// 275-282, 344-384).  dest [G][frames * channels]; what a read does not fill is zero.  counts [G]: READ_LATEST and
// READ the floats read, PEEK 1 when the newest frames were copied (0: fewer were available, nothing copied),
// AVAILABLE the frames available.
struct PubReadArgs
{
  const float* ring;  // instrument 0's ring of the signal
  uint32_t* state;    // [G][3] of the signal
  float* dest;
  int32_t* counts;
  int G, size, channels, mode, frames;
};

__global__ void __launch_bounds__(32 * kPubWarps) publish_read_kernel(const PubReadArgs a)
{
  const int g = blockIdx.x * kPubWarps + (threadIdx.x >> 5);
  if (g >= a.G) return;
  const int lane = threadIdx.x & 31;
  uint32_t* st = a.state + (size_t)g * 3;
  const uint32_t size = (uint32_t)a.size, dist = 2 * size - 1;
  const uint32_t w0 = st[0];
  uint32_t r = st[1];
  const uint32_t avail = (w0 - r) & dist;
  const uint32_t want = (uint32_t)a.frames * (uint32_t)a.channels;
  uint32_t n = 0, from = r;
  int32_t count = 0;
  if (a.mode == MLB_PUBLISHED_AVAILABLE)
    count = (int32_t)(avail / (uint32_t)a.channels);
  else if (a.mode == MLB_PUBLISHED_PEEK)
  {
    if (avail >= want) n = want, from = r + avail - want, count = 1;
  }
  else
  {
    uint32_t av = avail;
    if (a.mode == MLB_PUBLISHED_READ_LATEST && av > want) r = (r + (av - want)) & dist, av = want;  // discard
    n = av < want ? av : want;
    from = r, count = (int32_t)n;
    r = (r + n) & dist;
  }
  const float* ring = a.ring + (size_t)g * size;
  float* dst = a.dest ? a.dest + (size_t)g * want : nullptr;
  if (dst)
    for (uint32_t i = lane; i < want; i += 32) dst[i] = i < n ? ring[(from + i) & (size - 1)] : 0.f;
  __syncwarp();
  if (lane == 0)
  {
    if (a.counts) a.counts[g] = count;
    if (a.mode == MLB_PUBLISHED_READ_LATEST || a.mode == MLB_PUBLISHED_READ) st[1] = r;
  }
}

}  // namespace mlb
