"""The checker of the device router bank (api.RouterBank): G host routers (api.EventRouter, i.e. mlb::VoiceRouter, itself
pinned to the reference's EventsToSignals) driven from the same CSR input."""
import numpy as np

from madronalib_b200 import api, workloads as wl


def route_on_host(offsets, events, layout, mpe=False, unison=None, mod_cc=None):
    """offsets [T][G + 1] into events (api.EVENT_DTYPE) -> (records [T][V], change_offsets [T][G + 1], changes,
    overflow [G], unsupported [G]): per instrument g, one EventRouter gets block t's events at time t * 64 + frame and
    process_vector(t * 64).  A MIDI instrument of polyphony 0 has no records; its controller writes and unsupported
    count, which do not depend on routing state, come from a router of polyphony 1."""
    offsets = np.asarray(offsets)
    T, G = offsets.shape[0], offsets.shape[1] - 1
    V, poly, first = layout["n_voices"], layout["polyphony"], layout["first_voice"]
    rec = np.zeros((T, V), wl.VOICE_EVENTS_DTYPE)
    per = [[None] * G for _ in range(T)]
    overflow = np.zeros(G, np.int64)
    unsupported = np.zeros(G, np.int64)
    for g in range(G):
        P = int(poly[g])
        if P == 0 and mpe:
            raise ValueError("route_on_host: no host router of polyphony 0 in MPE")
        r = api.EventRouter(max(P, 1), api.EventRouter.MPE if mpe else api.EventRouter.MIDI,
                            unison=bool(unison[g]) if unison is not None else False)
        if mod_cc is not None:
            r.set_mod_cc(int(mod_cc[g]))
        buf = np.zeros(r.n_records, wl.VOICE_EVENTS_DTYPE)
        for t in range(T):
            for e in events[offsets[t, g]:offsets[t, g + 1]]:
                r.add_event(int(e["type"]), int(e["channel"]), int(e["source_idx"]), t * 64 + int(e["time"]),
                            float(e["value1"]), float(e["value2"]))
            n = r.process_vector(t * 64, buf)
            api.lib().mlb_router_clear_events(r._h)
            if P:
                overflow[g] += n
                rec[t, first[g]:first[g] + r.n_records] = buf
            per[t][g] = r.controller_changes()
        unsupported[g] = r.unsupported_events
        r.close()
    coff = np.zeros((T, G + 1), np.int32)
    chunks, n = [], 0
    for t in range(T):
        for g in range(G):
            coff[t, g] = n
            chunks.append(per[t][g])
            n += per[t][g].size
        coff[t, G] = n
    changes = np.concatenate(chunks) if chunks else np.zeros(0, api.CONTROLLER_CHANGE_DTYPE)
    return rec, coff, changes, overflow, unsupported


def csr(blocks, G):
    """blocks: per block t a dict {g: [(type, channel, source_idx, time, value1, value2), ...]} in arrival order
    -> (offsets [T][G + 1], events)."""
    T = len(blocks)
    offsets = np.zeros((T, G + 1), np.int32)
    rows = []
    for t, b in enumerate(blocks):
        for g in range(G):
            offsets[t, g] = len(rows)
            rows.extend(b.get(g, []))
        offsets[t, G] = len(rows)
    ev = np.zeros(len(rows), api.EVENT_DTYPE)
    for i, (ty, ch, src, tm, v1, v2) in enumerate(rows):
        ev[i] = (ty, ch, src, tm, np.float32(v1), np.float32(v2))
    return offsets, ev


ON, OFF, PEDAL, CC, BEND, NPRESS, CPRESS = 1, 4, 5, 6, 7, 8, 9
SPECIAL = [-0.0, float("inf"), -float("inf"), float("nan"), 1e-40, -1.4e-45]


def edge_blocks():
    """Hand-written blocks for the edge cases of one MIDI instrument of polyphony 2 (instrument 0) and one MPE-like
    keyed stream; used with both protocols."""
    return [
        # voice 0 in MIDI: two voices busy, a stolen note far (>= 128) from both keys goes to voice 0
        {0: [(ON, 1, 1, 3, 1.0, 0.5), (ON, 1, 2, 3, 1.0, 0.5), (ON, 1, 300, 5, 2.0, 0.7)]},
        # key numbers >= 128 index key states % 128; creator key unreduced
        {0: [(OFF, 1, 2, 0, 0.0, 0.0), (ON, 1, 130, 1, 3.0, 0.6), (OFF, 1, 130, 9, 0.0, 0.0)]},
        # pedal: note-offs during the pedal, release writes note-offs at time 0 after later events
        {0: [(PEDAL, 1, 0, 2, 1.0, 0.0), (ON, 1, 60, 4, 5.0, 0.8), (OFF, 1, 60, 10, 0.0, 0.0),
             (OFF, 1, 1, 11, 0.0, 0.0), (ON, 1, 61, 40, 5.1, 0.8), (PEDAL, 1, 0, 50, 0.0, 0.0)]},
        # special values copied by bits; equal time and type: the later arrival first
        {0: [(BEND, 1, 0, 7, SPECIAL[3], 0.0), (BEND, 1, 0, 7, SPECIAL[0], 0.0), (CC, 1, 1, 7, SPECIAL[1], 0.0),
             (CC, 1, 1, 7, SPECIAL[4], 0.0), (CC, 1, 74, 8, SPECIAL[5], 0.0), (CPRESS, 1, 0, 9, SPECIAL[2], 0.0),
             (NPRESS, 1, 61, 9, SPECIAL[3], 0.0), (CC, 1, 200, 9, 0.25, 0.0), (CC, 1, 120, 9, 0.0, 0.0)]},
        # CC 123 writes note-offs to all 17 voices
        {0: [(ON, 1, 62, 1, 5.2, 0.9), (CC, 1, 123, 20, -0.0, 0.0), (ON, 1, 63, 30, 5.3, 0.9)]},
        # ignored types
        {0: [(0, 1, 1, 1, 1.0, 1.0), (2, 1, 60, 2, 1.0, 1.0), (3, 1, 60, 3, 1.0, 1.0), (10, 1, 5, 4, 1.0, 1.0)]},
    ]


def unison_release_blocks():
    """Unison: the first note (note-on index 0) is still held when the later one is released: strict > from 0 never
    picks index 0, so the fall-back key is key 0 (whose pitch is 0); then a third note makes the fall-back real."""
    return [
        {0: [(ON, 1, 50, 1, 4.0, 0.5)]},
        {0: [(ON, 1, 55, 1, 4.5, 0.6)]},
        {0: [(OFF, 1, 55, 2, 0.0, 0.0)]},
        {0: [(ON, 1, 57, 1, 4.7, 0.6), (ON, 1, 59, 2, 4.9, 0.6)]},
        {0: [(OFF, 1, 59, 3, 0.0, 0.0)]},
        {0: [(OFF, 1, 57, 3, 0.0, 0.0), (OFF, 1, 50, 5, 0.0, 0.0)]},
    ]
