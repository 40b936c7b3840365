// router_kernel.cuh -- K12: the event routing of EventsToSignals (source/app/MLEventsToSignals.cpp:352-418, 476-960) for
// G instruments at once, exactly as mlb::VoiceRouter (include/mlb200_events.hpp) routes one: voice allocation (the
// rotating free-voice search, stealing by nearest key), unison, the sustain pedal, MPE channels and CC 123.
//
// Input per block t: the events of instrument g are events[offsets[t][g] .. offsets[t][g + 1]) in arrival (addEvent)
// order, Event::time the frame within the block (0..63).  Output per block: the mlb_voice_events record of every voice
// (the buffer K7 reads), and the controller writes as a CSR change list (change_offsets [T][G + 1] into changes) that
// K11 consumes as it stands.
//
// Three launches per call:
//   router_count_kernel   one CTA per block: each instrument's controller writes are counted (whether an event writes a
//                         controller depends on its type and the protocol only, never on routing state) and scanned over
//                         the instruments: change_offsets[t][g] = the block-local start, change_offsets[t][G] = the
//                         block's total.  The records of voices of no instrument are zeroed here.
//   router_bank_kernel    one warp per instrument, walking the blocks in order with the whole routing state in
//                         registers: lane v mirrors voice v (0..16) and keeps its record in shared memory, lane l owns
//                         keys 4l..4l+3.  Events are taken in addEvent's order -- by (time, type), and the later arrival
//                         first among equals -- by a warp arg-min per event, so any number of events per block works.
//                         The free-voice search, the nearest-voice search, the held-note count and the unison arg-max
//                         are ballots and warp reductions.  Each block's records leave as coalesced warp stores, and the
//                         warp turns its change offsets into global ones by adding the totals of the earlier blocks.
//   router_total_kernel   one CTA: change_offsets[t][G] = the inclusive sum of the block totals.
// No allocation, atomics or synchronisation: a call can be captured into a CUDA graph.  State between calls is
// kRouterWords coalesced words per lane and instrument.
#pragma once
#include <cub/block/block_scan.cuh>

#include "voice_kernel.cuh"

namespace mlb
{
constexpr int kRouterWarps = 4;           // instruments per 128-thread CTA of router_bank_kernel
constexpr int kRouterScanThreads = 512;   // threads of the count and total CTAs
constexpr int kRouterWords = 16;          // state words per lane and instrument
constexpr int kRouterVoices = 17;         // EventsToSignals::kMaxVoices + the main voice
constexpr int kRecordWords = sizeof(mlb_voice_events) / 4;
static_assert(sizeof(mlb_voice_events) == 72 && sizeof(mlb_event) == 16, "record layouts");

// state word w of lane l of instrument g: state[(g * kRouterWords + w) * 32 + l]
enum RouterWord
{
  RW_KEY_STATE = 0,   // 4 words: KeyState::state of key 4l + s (0 off, 1 on, 2 sustained)
  RW_KEY_PITCH = 4,   // 4 words: KeyState::pitch (float bits)
  RW_KEY_INDEX = 8,   // 4 words: KeyState::noteOnIndex
  RW_CREATOR = 12,    // lanes 0..16: Voice::creatorKeyIdx
  RW_VELOCITY = 13,   // lanes 0..16: Voice::currentVelocity (float bits)
  RW_OVERFLOW = 14,   // lanes 0..16: note events of this voice that found its record full, since creation
  RW_SCALAR = 15      // one scalar per lane (RouterScalar)
};
enum RouterScalar { RS_LAST_FREE = 0, RS_PEDAL, RS_NOTE_ON_INDEX, RS_UNSUPPORTED };
enum RouterInst { RI_POLY = 0, RI_FIRST, RI_UNISON, RI_MOD_CC, RI_COUNT };  // settings table [RI_COUNT][G]
enum { KEY_OFF = 0, KEY_ON = 1, KEY_SUSTAINED = 2 };

struct RouterArgs
{
  const int32_t* offsets;          // [T][G + 1] into events
  const mlb_event* events;         // arrival order
  mlb_voice_events* records;       // [T][V]
  int32_t* change_offsets;         // [T][G + 1] into changes
  mlb_controller_change* changes;
  uint32_t* state;                 // [G][kRouterWords][32]
  const int32_t* inst;             // [RI_COUNT][G]
  const int32_t* unowned;          // [n_unowned] voices of no instrument
  int n_unowned, G, V, T, mpe;
};

// a controller event, and channel pressure in the MIDI protocol, write one SmoothedController inputValue
__host__ __device__ inline bool router_writes_controller(int type, int mpe) { return type == 6 || (type == 9 && !mpe); }

__global__ void __launch_bounds__(kRouterScanThreads) router_count_kernel(RouterArgs a)
{
  using Scan = cub::BlockScan<int, kRouterScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int t = blockIdx.x;
  const int32_t* off = a.offsets + (size_t)t * (a.G + 1);
  int32_t* coff = a.change_offsets + (size_t)t * (a.G + 1);
  int carry = 0;
  for (int g0 = 0; g0 < a.G; g0 += kRouterScanThreads)
  {
    const int g = g0 + (int)threadIdx.x;
    int n = 0;
    if (g < a.G)
      for (int i = off[g]; i < off[g + 1]; ++i) n += router_writes_controller(a.events[i].type, a.mpe);
    int start, total;
    Scan(tmp).ExclusiveSum(n, start, total);
    if (g < a.G) coff[g] = carry + start;
    carry += total;
    __syncthreads();  // tmp is reused
  }
  if (threadIdx.x == 0) coff[a.G] = carry;
  uint32_t* rec = reinterpret_cast<uint32_t*>(a.records + (size_t)t * a.V);
  for (int i = threadIdx.x; i < a.n_unowned * kRecordWords; i += blockDim.x)
    rec[(size_t)a.unowned[i / kRecordWords] * kRecordWords + i % kRecordWords] = 0u;
}

__global__ void __launch_bounds__(kRouterScanThreads) router_total_kernel(int32_t* change_offsets, int G, int T)
{
  using Scan = cub::BlockScan<int, kRouterScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int t0 = 0; t0 < T; t0 += kRouterScanThreads)
  {
    const int t = t0 + (int)threadIdx.x;
    int32_t* p = change_offsets + (size_t)t * (G + 1) + G;
    int end, total;
    Scan(tmp).InclusiveSum(t < T ? *p : 0, end, total);
    if (t < T) *p = carry + end;
    carry += total;
    __syncthreads();
  }
}

// mlb_routers_clear: every state word back to 0 (VoiceRouter's constructor), the counter words kept
__global__ void router_clear_kernel(uint32_t* state, size_t n_words)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_words; i += (size_t)gridDim.x * blockDim.x)
  {
    const int w = (int)(i / 32 % kRouterWords), l = (int)(i % 32);
    if (w != RW_OVERFLOW && !(w == RW_SCALAR && l == RS_UNSUPPORTED)) state[i] = 0u;
  }
}

__global__ void __launch_bounds__(32 * kRouterWarps) router_bank_kernel(RouterArgs a)
{
  constexpr unsigned kAll = 0xFFFFFFFFu;
  __shared__ mlb_voice_events stage_all[kRouterWarps][kRouterVoices];
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * kRouterWarps + (threadIdx.x >> 5);
  if (g >= a.G) return;  // the whole warp
  mlb_voice_events* stage = stage_all[threadIdx.x >> 5];
  uint32_t* stage_w = reinterpret_cast<uint32_t*>(stage);
  const int P = a.inst[RI_POLY * a.G + g], first = a.inst[RI_FIRST * a.G + g];
  const bool unison = a.inst[RI_UNISON * a.G + g] != 0;
  const int mod_cc = a.inst[RI_MOD_CC * a.G + g];
  const bool mpe = a.mpe != 0;
  const int n_rec = mpe ? P + 1 : P;
  const bool is_voice = lane < kRouterVoices;
  const bool in_poly = lane >= 1 && lane <= P;              // voices 1..polyphony
  const bool has_rec = lane <= P && lane >= (mpe ? 0 : 1);  // MIDI: the main voice has no record
  const int slot = mpe ? lane : lane - 1;

  uint32_t* st = a.state + (size_t)g * kRouterWords * 32 + lane;
  uint32_t ks[4], ki[4];
  float kp[4];
#pragma unroll
  for (int s = 0; s < 4; ++s)
  {
    ks[s] = st[(RW_KEY_STATE + s) * 32];
    kp[s] = __uint_as_float(st[(RW_KEY_PITCH + s) * 32]);
    ki[s] = st[(RW_KEY_INDEX + s) * 32];
  }
  int ck = (int)st[RW_CREATOR * 32];
  float vel = __uint_as_float(st[RW_VELOCITY * 32]);
  uint32_t overflow = st[RW_OVERFLOW * 32];
  const uint32_t sc = st[RW_SCALAR * 32];
  int last_free = (int)__shfl_sync(kAll, sc, RS_LAST_FREE);
  bool pedal = __shfl_sync(kAll, sc, RS_PEDAL) != 0;
  uint32_t note_on_index = __shfl_sync(kAll, sc, RS_NOTE_ON_INDEX);
  uint32_t unsupported = __shfl_sync(kAll, sc, RS_UNSUPPORTED);

  int rn = 0;          // n_events of this lane's record
  uint32_t rmask = 0;  // set_mask of this lane's record
  // Voice::writeNoteEvent as seen from the router, on the lanes `me`: mirror, then append to the record
  auto note = [&](bool me, int type, int time, float v1, float v2, int key, bool glide, bool reset)
  {
    if (!me) return;
    if (type == MLB_EV_NOTE_ON || type == MLB_EV_NOTE_RETRIG)
      ck = key, vel = v2;
    else if (type == MLB_EV_NOTE_OFF)
      ck = 0, vel = 0.f;
    else
      return;
    if (!has_rec) return;
    if (rn >= MLB_VOICE_MAX_EVENTS)
    {
      ++overflow;
      return;
    }
    mlb_voice_events& r = stage[slot];
    r.time[rn] = (uint8_t)min(max(time, 0), MLB_BLOCK);
    r.type[rn] = (uint8_t)type;
    r.flags[rn] = (uint8_t)((glide ? MLB_EVF_GLIDE : 0) | (reset ? MLB_EVF_RESET : 0));
    r.value1[rn] = v1;
    r.value2[rn] = v2;
    ++rn;
  };
  auto set_current = [&](bool me, unsigned bit, float v)
  {
    if (!me) return;
    mlb_voice_events& r = stage[slot];
    rmask |= bit;
    switch (bit)
    {
      case MLB_SET_BEND: r.bend = v; break;
      case MLB_SET_MOD: r.mod = v; break;
      case MLB_SET_X: r.x = v; break;
      case MLB_SET_Y: r.y = v; break;
      case MLB_SET_Z: r.z = v; break;
      default: r.pressure = v; break;
    }
  };
  auto held_notes = [&]()
  {
    int n = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) n += ks[s] == KEY_ON;
    return (int)__reduce_add_sync(kAll, (unsigned)n);
  };
  // KeyState::state of key k (0..127), on every lane that asks for its own k
  auto key_state_of = [&](int k)
  {
    uint32_t r = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s)
    {
      const uint32_t x = __shfl_sync(kAll, ks[s], k >> 2);
      if ((k & 3) == s) r = x;
    }
    return r;
  };

  int base = 0;  // controller writes of the earlier blocks
#pragma unroll 1
  for (int t = 0; t < a.T; ++t)
  {
    const size_t row = (size_t)t * (a.G + 1);
    for (int i = lane; i < n_rec * kRecordWords; i += 32) stage_w[i] = 0u;
    __syncwarp();
    rn = 0, rmask = 0;
    const int o0 = a.offsets[row + g], o1 = a.offsets[row + g + 1];
    const int cstart = base + a.change_offsets[row + g];
    int cpos = cstart;
    uint32_t prev_hi = 0, prev_lo = 0;
#pragma unroll 1
    for (int k = 0; k < o1 - o0; ++k)
    {
      // the next event in addEvent's order: the smallest (time << 8 | type, ~arrival) above the previous one
      uint32_t best_hi = kAll, best_lo = kAll;
      for (int j = o0 + lane; j < o1; j += 32)
      {
        const uint2 h = __ldg(reinterpret_cast<const uint2*>(a.events + j));
        const uint32_t hi = (h.y << 8) | (h.x & 0xFFu), lo = ~(uint32_t)(j - o0);
        const bool after = k == 0 || hi > prev_hi || (hi == prev_hi && lo > prev_lo);
        if (after && (hi < best_hi || (hi == best_hi && lo < best_lo))) best_hi = hi, best_lo = lo;
      }
      prev_hi = __reduce_min_sync(kAll, best_hi);
      prev_lo = __reduce_min_sync(kAll, best_hi == prev_hi ? best_lo : kAll);
      const uint4 e = __ldg(reinterpret_cast<const uint4*>(a.events + o0 + (int)~prev_lo));
      const int type = (int)(e.x & 0xFFu), ch = (int)((e.x >> 8) & 0xFFu), src = (int)(e.x >> 16), time = (int)e.y;
      const float v1 = __uint_as_float(e.z), v2 = __uint_as_float(e.w);
      const int key = mpe ? ch : src;  // getKeyIndex
      switch (type)
      {
        case 1:  // noteOn, .cpp:513-553
        {
          const int kk = key & 127;
#pragma unroll
          for (int s = 0; s < 4; ++s)
          {
            // selects, not an indexed store: the key arrays stay in registers
            const bool hit = lane == kk >> 2 && s == (kk & 3);
            ks[s] = hit ? (uint32_t)KEY_ON : ks[s];
            ki[s] = hit ? note_on_index : ki[s];
            kp[s] = hit ? v1 : kp[s];
          }
          ++note_on_index;
          if (unison)
          {
            const bool first_note = held_notes() == 1;
            note(in_poly, MLB_EV_NOTE_ON, time, v1, v2, key, !first_note, first_note);
            break;
          }
          const unsigned free = __ballot_sync(kAll, in_poly && ck == 0);
          if (free)  // findFreeVoice: the first free voice after lastFreeVoiceFound_, wrapping to voice 1
          {
            const unsigned later = free & ~((2u << last_free) - 1u);
            last_free = __ffs(later ? later : free) - 1;
            note(lane == last_free, MLB_EV_NOTE_ON, time, v1, v2, key, true, true);
          }
          else  // findNearestVoice(sourceIdx): the first voice at the least distance below 128, else voice 0
          {
            const unsigned d = (unsigned)abs(src - ck);
            const unsigned m = __reduce_min_sync(kAll, in_poly && d < 128u ? (d << 5) | (unsigned)lane : kAll);
            note(lane == (m == kAll ? 0 : (int)(m & 31u)), MLB_EV_NOTE_RETRIG, time, v1, v2, key, true, true);
          }
          break;
        }
        case 4:  // noteOff, .cpp:555-628
        {
          const int kk = key & 127;
#pragma unroll
          for (int s = 0; s < 4; ++s)
            ks[s] = lane == kk >> 2 && s == (kk & 3) ? (uint32_t)(pedal ? KEY_SUSTAINED : KEY_OFF) : ks[s];
          if (unison)
          {
            if (held_notes() == 0)
              note(in_poly, MLB_EV_NOTE_OFF, time, v1, v2, 0, true, true);
            else if (key == __shfl_sync(kAll, ck, 1))
            {
              // fall back to the most recently played key still held: strict > from 0 over the keys in order
              const float vel1 = __shfl_sync(kAll, vel, 1);
              uint32_t bi = 0;
              int bk = 0;
#pragma unroll
              for (int s = 0; s < 4; ++s)
                if (ks[s] == KEY_ON && ki[s] > bi) bi = ki[s], bk = 4 * lane + s;
              const uint32_t mx = __reduce_max_sync(kAll, bi);
              const unsigned at = __ballot_sync(kAll, bi == mx);
              const int recent = __shfl_sync(kAll, bk, __ffs(at) - 1);
              const int rk = mx > 0 ? recent : 0;
              // one shuffle per slot, then a select: an indexed read kp[rk & 3] would put kp in local memory
              float pitch = 0.f;
#pragma unroll
              for (int s = 0; s < 4; ++s)
              {
                const float x = __shfl_sync(kAll, kp[s], rk >> 2);
                if ((rk & 3) == s) pitch = x;
              }
              note(in_poly, MLB_EV_NOTE_ON, time, pitch, vel1, rk, true, true);
            }
            break;
          }
          if (!pedal) note(in_poly && ck == key, MLB_EV_NOTE_OFF, time, v1, v2, key, true, true);
          break;
        }
        case 5:  // sustainPedal, .cpp:823-841: the release writes note-offs at time 0
        {
          pedal = v1 > 0.5f;
          if (!pedal)
          {
            const bool held = key_state_of(ck & 127) == KEY_SUSTAINED;
            note(in_poly && held, MLB_EV_NOTE_OFF, 0, 0.f, 0.f, 0, true, true);
          }
          break;
        }
        case 6:  // controller, .cpp:737-820
        {
          const int ctrl = min(src, 128);
          if (lane == 0)
            *reinterpret_cast<uint2*>(a.changes + cpos) = make_uint2((uint32_t)ctrl, __float_as_uint(v1));
          ++cpos;
          if (ctrl == 128 && !mpe) set_current(in_poly, MLB_SET_PRESSURE, v1);
          if (ctrl == 120)
          {
            if (v1 == 0.f) ++unsupported;  // all sound off: counted, not routed
          }
          else if (ctrl == 123)
          {
            if (v1 == 0.f) note(is_voice, MLB_EV_NOTE_OFF, time, v1, v2, 0, false, true);  // all 17 voices
          }
          else
          {
            const bool me = in_poly && (!mpe || ck == ch);
            if (ctrl == mod_cc) set_current(me, MLB_SET_MOD, v1);
            if (ctrl == 73)
              set_current(me, MLB_SET_X, v1);
            else if (ctrl == 74)
              set_current(me, MLB_SET_Y, v1);
          }
          break;
        }
        case 7:  // pitch bend, .cpp:700-735
          if (!mpe)
            set_current(in_poly, MLB_SET_BEND, v1);
          else if (ch == 1)
            set_current(lane == 0, MLB_SET_BEND, v1);
          else if (ch != 0)
            set_current(in_poly && ck == ch, MLB_SET_BEND, v1);
          break;
        case 8:  // note pressure, .cpp:673-697; ignored in MPE
          if (!mpe) set_current(in_poly && ck == src, MLB_SET_Z, v1);
          break;
        case 9:  // channel pressure, .cpp:634-670
          if (!mpe)
          {
            if (lane == 0)
              *reinterpret_cast<uint2*>(a.changes + cpos) = make_uint2(128u, __float_as_uint(v1));
            ++cpos;
            set_current(in_poly, MLB_SET_PRESSURE, v1);
          }
          else if (ch == 1)
            set_current(lane == 0, MLB_SET_Z, v1);
          else if (ch != 0)
            set_current(in_poly && ck == ch, MLB_SET_Z, v1);
          break;
        default: break;  // null, retrigger, sustain, program change: ignored
      }
    }
    __syncwarp();  // every lane has read change_offsets[row + g] before lane 0 overwrites it
    if (lane == 0) a.change_offsets[row + g] = cstart;
    base += a.change_offsets[row + a.G];  // the block's total (router_total_kernel makes it global afterwards)
    if (has_rec) stage[slot].n_events = (uint8_t)rn, stage[slot].set_mask = (uint8_t)rmask;
    __syncwarp();
    uint32_t* dst = reinterpret_cast<uint32_t*>(a.records + (size_t)t * a.V + first);
    for (int i = lane; i < n_rec * kRecordWords; i += 32) dst[i] = stage_w[i];
    __syncwarp();
  }

#pragma unroll
  for (int s = 0; s < 4; ++s)
  {
    st[(RW_KEY_STATE + s) * 32] = ks[s];
    st[(RW_KEY_PITCH + s) * 32] = __float_as_uint(kp[s]);
    st[(RW_KEY_INDEX + s) * 32] = ki[s];
  }
  st[RW_CREATOR * 32] = (uint32_t)ck;
  st[RW_VELOCITY * 32] = __float_as_uint(vel);
  st[RW_OVERFLOW * 32] = overflow;
  st[RW_SCALAR * 32] = lane == RS_LAST_FREE ? (uint32_t)last_free
                       : lane == RS_PEDAL ? (uint32_t)pedal
                       : lane == RS_NOTE_ON_INDEX ? note_on_index
                       : lane == RS_UNSUPPORTED ? unsupported
                                                : 0u;
}

}  // namespace mlb
