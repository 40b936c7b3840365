"""Event phrases for the smoothed-controller tests (tests/test_controllers.py, tests/test_gpu_controllers.py) and the
golden writer (tests/golden/make_controllers_golden.py)."""
from __future__ import annotations

import numpy as np

CONTROLLER, CHANNEL_PRESSURE, NOTE_ON, NOTE_OFF = 6, 9, 1, 4
ALL_CONTROLLERS = list(range(129))
SAMPLE_RATES = (44100.0, 48000.0, 96000.0)
GLIDE_VECTORS = {44100.0: 13, 48000.0: 14, 96000.0: 29}  # int(int(sr * 0.02f) / 64): 881, 959, 1919 samples

_SPECIAL = np.array([0.0, -0.0, 1.0, 0.5, -0.75, np.inf, -np.inf, np.nan, 1e-40, -1e-42, 1.4e-45, 3e38, -3e38,
                     0.1, 1.0 / 127], np.float32)


def special_phrases(n_instruments: int, n_blocks: int, seed: int, n_events: int = 24):
    """Per instrument a list of (type, channel, source_idx, time, value1, value2): controller writes (numbers 0..128,
    above 128, CC 120 and 123), channel pressure and notes, values from -0, +-inf, NaN, subnormals and ordinary
    numbers, several writes to one controller at one time, glides interrupted by new targets.  CC 120 is never 0:
    "all sound off" clears the reference's event buffer in mid-vector (MLEventsToSignals.cpp:746-753), which the
    project does not model."""
    rng = np.random.default_rng(seed)
    numbers = np.array([0, 1, 7, 11, 64, 74, 120, 123, 127, 128, 129, 300, 65535], np.int64)
    phrases = []
    for g in range(n_instruments):
        evs = []
        for _ in range(int(rng.integers(0, n_events + 1))):
            time = int(rng.integers(0, n_blocks * 64))
            if rng.random() < 0.3:  # a burst at one instant: the last one added to one controller is applied first
                time = evs[-1][3] if evs else time
            value = float(_SPECIAL[rng.integers(0, len(_SPECIAL))]) if rng.random() < 0.4 else \
                float(np.float32(rng.integers(0, 128) / 127))
            r = rng.random()
            if r < 0.7:
                number = int(numbers[rng.integers(0, len(numbers))])
                if number == 120 and value == 0:  # "all sound off" empties the reference's event buffer: out of scope
                    value = 0.5
                evs.append((CONTROLLER, int(rng.integers(1, 17)), number, time, value, 0.0))
            elif r < 0.85:
                evs.append((CHANNEL_PRESSURE, int(rng.integers(1, 17)), 0, time, value, 0.0))
            else:
                evs.append((NOTE_ON if rng.random() < 0.5 else NOTE_OFF, 1, int(rng.integers(36, 90)), time,
                            float(rng.integers(36, 90)), 0.8))
        phrases.append(evs)
    return phrases
