"""The project's counter-based random draws restated in integer arithmetic (NumPy uint32 / int64, no torch), from csrc/render.cu
(hash_uniform, the sampler's seed conventions in k_sample) and csrc/select.cu (mix32, point_key, k_select_rays' per-scan seed and
top-N selection), plus the per-iteration seed streams of the captured loops.

Every function takes Python ints or NumPy arrays and returns NumPy arrays of the kernel's type, so a kernel's output can be compared
with these bit for bit.  Seeds travel through the API as int32 device words; `u32` / `i32` convert between the two views."""
import numpy as np

M32 = 0xFFFFFFFF
GOLDEN_SEL = 0x9E3779B9             # k_select_rays: per-scan seed mix32(seed ^ GOLDEN_SEL * (f + 1))
SEED_INC_SELECT = 0x632BE5          # per-iteration advance of the ray-selection seed of every captured loop
SEED_INC_NOISE = 0x3779B1           # per-iteration advance of the sampler-noise seed
U_LO, U_HI = np.float32(0.001), np.float32(0.999)      # hash_uniform's clamp (voxel_helpers.py:301)


def u32(x):
    """The uint32 view of a seed given as a Python int or an int32 / int64 word (int32 -1 -> 0xFFFFFFFF)."""
    a = np.asarray(x)
    if a.dtype.kind != "u":
        a = a.astype(np.int64)          # int32 / int64 words and Python ints below 2^63: two's complement carries over
    return a.astype(np.uint64) & np.uint64(M32)


def i32(x):
    """The int32 word holding a seed given as any integer (its value modulo 2^32): what a device seed tensor stores."""
    return (np.asarray(x, dtype=np.int64) & M32).astype(np.uint32).view(np.int32)


def _mul(a, b):
    """(a * b) mod 2^32 of uint32 operands, in uint64 so nothing overflows."""
    return (np.asarray(a, np.uint64) * np.uint64(b)) & np.uint64(M32)


def mix32(x):
    """csrc/select.cu mix32 (and the finaliser inside hash_uniform): xor-shift / multiply, all mod 2^32."""
    x = u32(x)
    x = x ^ (x >> np.uint64(16))
    x = _mul(x, 0x7FEB352D)
    x = x ^ (x >> np.uint64(15))
    x = _mul(x, 0x846CA68B)
    x = x ^ (x >> np.uint64(16))
    return x.astype(np.uint32)


def scan_seed(seed, f=0, batched=False):
    """k_select_rays' seed of scan f: mix32(seed ^ 0x9E3779B9 (f + 1)).  nl_select_rays_batch draws every problem as frame 0 of a
    one-scan call (f = 0 whatever its index), with its own seed."""
    ff = 0 if batched else int(f)
    return mix32(u32(seed) ^ _mul(ff + 1, GOLDEN_SEL))


def point_key(seed, f, i, batched=False):
    """The 32-bit key of point i of scan f: mix32(scan_seed ^ mix32(i * 0x9E3779B1 + 0x7F4A7C15))."""
    s = np.uint64(scan_seed(seed, f, batched))
    inner = mix32((_mul(i, 0x9E3779B1) + np.uint64(0x7F4A7C15)) & np.uint64(M32))
    return mix32(s ^ inner.astype(np.uint64))


def top_n(keys, N):
    """Indices of the N smallest keys, ties to the lower index, in point order (k_select_rays' subset, emitted in point order)."""
    keys = np.asarray(keys, np.uint32)
    N = min(int(N), keys.shape[0])
    order = np.lexsort((np.arange(keys.shape[0]), keys))      # by key, then by index
    return np.sort(order[:N])


def hash_word(seed, ray, step):
    """hash_uniform's 32-bit word before the float conversion: mix32(seed ^ ray 0x9E3779B1 ^ step 0x85EBCA77)."""
    x = u32(seed) ^ _mul(ray, 0x9E3779B1) ^ _mul(step, 0x85EBCA77)
    return mix32(x)


def hash_uniform(seed, ray, step, clamp=True):
    """csrc/render.cu hash_uniform: (x >> 8) / 2^24 in float32 (exact: 24 bits), clamped to [0.001, 0.999]."""
    u = (hash_word(seed, ray, step) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return np.minimum(np.maximum(u, U_LO), U_HI) if clamp else u


def sampler_seed(rng_seed=0, rng_seed_dev=None, seg_seed=None):
    """The seed k_sample hashes with: a host seed as given (0: no hash, every noise value is the midpoint 0.5); a device seed or a
    batched problem's seed with 0 replaced by 1.  Returns the uint32 seed, 0 meaning "midpoints"."""
    if seg_seed is not None:
        s = int(u32(seg_seed))
        return s if s else 1
    if rng_seed_dev is not None:
        s = int(u32(rng_seed_dev))
        return s if s else 1
    return int(u32(rng_seed))


def noise_by_ray(seed, n_rays, n_steps):
    """f32[n_rays, n_steps]: the noise k_sample draws for ray r (its index within its problem) at stratum i."""
    if seed == 0:
        return np.full((n_rays, n_steps), 0.5, np.float32)
    r = np.arange(n_rays, dtype=np.uint64)[:, None]
    i = np.arange(n_steps, dtype=np.uint64)[None, :]
    return hash_uniform(seed, r, i)


def noise_table(seed, hit_rank, n_steps):
    """The restated draws laid out the way k_sample reads a noise tensor: row q (hit rank) holds the noise of the ray whose hit
    rank is q, although the hash is keyed by that ray's index r.  hit_rank: i32[R] of one problem (-1 for a miss, else its rank).
    Returns f32[max(R_hit, 1), n_steps]."""
    hit_rank = np.asarray(hit_rank)
    rays = np.flatnonzero(hit_rank >= 0)
    out = np.zeros((max(rays.shape[0], 1), n_steps), np.float32)
    if seed == 0:
        out[hit_rank[rays]] = 0.5
    else:
        out[hit_rank[rays]] = hash_uniform(seed, rays.astype(np.uint64)[:, None], np.arange(n_steps, dtype=np.uint64)[None, :])
    return out


def seed_at(s0, inc, t):
    """A seed stream advanced by `inc` t times, modulo 2^32 (uint32)."""
    return np.uint32((int(u32(s0)) + int(inc) * int(t)) & M32)
