"""Inputs shared by the per-instrument bus tests (K10) and tests/golden/make_buses_golden.py."""
import numpy as np

# a bus layout over GOLDEN_V voices with counts 0, 1, 3 and 16, gaps (voices 4, 8, 36-38 are in no bus) and overlaps
GOLDEN_V = 40
GOLDEN_FIRST = np.array([0, 0, 5, 9, 20, 21, 30, 39, 1], np.int32)
GOLDEN_COUNT = np.array([0, 1, 3, 16, 16, 4, 3, 1, 3], np.int32)


def special_rows(T: int, P: int, V: int, seed: int, nonfinite: bool = True) -> np.ndarray:
    """[T][P][V][64] f32 voice rows: normals of several scales, with -0, +-inf, NaN, subnormals and cancelling large
    magnitudes (+-3e38 overflows when two meet, +-1e30 cancels) scattered in, plus whole rows of -0 and of
    subnormals.  nonfinite=False leaves out +-inf, NaN and +-3e38, so that sums over thousands of voices stay finite."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((T, P, V, 64)) * 10.0 ** rng.integers(-3, 4, (T, P, V, 1))).astype(np.float32)
    kind = rng.integers(0, 1000, x.shape)
    sign = np.where(rng.random(x.shape) < 0.5, -1.0, 1.0).astype(np.float32)
    x[kind < 60] = -0.0
    sub = (kind >= 60) & (kind < 160)
    x[sub] = (rng.uniform(-1, 1, int(sub.sum())) * 1e-38).astype(np.float32)
    if nonfinite:
        x[(kind >= 160) & (kind < 200)] = (sign * np.float32(3e38))[(kind >= 160) & (kind < 200)]
    x[(kind >= 200) & (kind < 260)] = (sign * np.float32(1e30))[(kind >= 200) & (kind < 260)]
    if nonfinite:
        x[kind == 260] = np.inf
        x[kind == 261] = -np.inf
        x[kind == 262] = np.nan
    x[:, :, ::7] = -0.0
    x[:, :, 3::11] = (rng.uniform(-1, 1, x[:, :, 3::11].shape) * 1e-39).astype(np.float32)
    return x


def random_layout(rng, V: int, G: int, max_count: int):
    """G random ranges of the V voices with counts in [0, max_count] (gaps and overlaps arise at random)."""
    count = rng.integers(0, min(max_count, V) + 1, G).astype(np.int32)
    first = np.array([rng.integers(0, V - c + 1) for c in count], np.int32)
    return first, count
