"""NumPy reference of the lossy checkpoint codec (the TurboQuant file of the reference's include/statevector_turboquant.hpp),
bit for bit in plain sequential IEEE arithmetic:
  - mt19937_64 vectorised in uint64 (the C++ standard's engine);
  - std::normal_distribution<real> as GCC 13's bits/random.tcc implements it: the polar method with the second value saved,
    uniforms from generate_canonical<real> (one 64-bit draw, real(x) / 2^64, clamped below 1 with nextafter(1, 0)), and log
    from the C library (logf / log through ctypes: the function the reference calls);
  - modified Gram-Schmidt, the rotations and the scale as sequential loops over j in `real`, vectorised across outputs.
"""
import ctypes
import ctypes.util

import numpy as np

_LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
_LIBM.logf.argtypes, _LIBM.logf.restype = [ctypes.c_float], ctypes.c_float
_LIBM.log.argtypes, _LIBM.log.restype = [ctypes.c_double], ctypes.c_double

_N, _M = 312, 156
_A = np.uint64(0xB5026F5AA96619E9)
_UM, _LM = np.uint64(0xFFFFFFFF80000000), np.uint64(0x7FFFFFFF)


class MT19937_64:
    """std::mt19937_64; draw(k) returns the next k outputs."""

    def __init__(self, seed=5489):
        mt = np.zeros(_N, dtype=np.uint64)
        mt[0] = np.uint64(seed)
        with np.errstate(over="ignore"):
            for i in range(1, _N):
                prev = int(mt[i - 1])
                mt[i] = np.uint64((6364136223846793005 * (prev ^ (prev >> 62)) + i) & 0xFFFFFFFFFFFFFFFF)
        self.mt, self.idx = mt, _N

    def _twist(self):
        mt = self.mt

        def upd(cur, nxt, far):
            y = (cur & _UM) | (nxt & _LM)
            return far ^ (y >> np.uint64(1)) ^ np.where((y & np.uint64(1)) != 0, _A, np.uint64(0))

        mt[0:_N - _M] = upd(mt[0:_N - _M], mt[1:_N - _M + 1], mt[_M:_N])
        mt[_N - _M:_N - 1] = upd(mt[_N - _M:_N - 1], mt[_N - _M + 1:_N], mt[0:_M - 1])
        mt[_N - 1:_N] = upd(mt[_N - 1:_N], mt[0:1], mt[_M - 1:_M])
        self.idx = 0

    def draw(self, k):
        out = []
        while k:
            if self.idx == _N:
                self._twist()
            take = min(k, _N - self.idx)
            y = self.mt[self.idx:self.idx + take].copy()
            self.idx += take
            k -= take
            y ^= (y >> np.uint64(29)) & np.uint64(0x5555555555555555)
            y ^= (y << np.uint64(17)) & np.uint64(0x71D67FFFEDA60000)
            y ^= (y << np.uint64(37)) & np.uint64(0xFFF7EEE000000000)
            y ^= y >> np.uint64(43)
            out.append(y)
        return np.concatenate(out) if out else np.zeros(0, dtype=np.uint64)


def _canonical(x, real):
    """generate_canonical<real, digits>(mt19937_64) for the draws x"""
    u = x.astype(real) * real(2.0 ** -64)
    return np.where(u >= real(1), np.nextafter(real(1), real(0)), u).astype(real)


def normals(seed, count, real):
    """the first `count` values of std::normal_distribution<real>(0, 1) over std::mt19937_64(seed)"""
    real = np.dtype(real).type
    rng = MT19937_64(seed)
    log = _LIBM.logf if real is np.float32 else _LIBM.log
    out = []
    while len(out) < count:
        # attempts in order; the generator is never used after the last value, so a batch may overshoot
        want = (count - len(out)) + 64
        u = _canonical(rng.draw(2 * want), real).reshape(want, 2)
        # result_type(2.0) * u - 1.0: the product in real, the difference in double, rounded back to real
        xy = ((real(2) * u).astype(np.float64) - 1.0).astype(real)
        x, y = xy[:, 0], xy[:, 1]
        r2 = x * x + y * y
        for a in np.flatnonzero(~((r2.astype(np.float64) > 1.0) | (r2 == 0))):
            r = r2[a]
            mult = np.sqrt(real(-2) * real(log(r)) / r)
            out += [y[a] * mult, x[a] * mult]  # the first call returns y * mult and saves x * mult
    v = np.array(out[:count], dtype=real)
    return v * real(1) + real(0)


def rotation(d, seed, real):
    """the d x d rotation of `seed`, column-major flattened (R[j d + i] = row i of column j)"""
    real = np.dtype(real).type
    R = normals(seed, d * d, real).reshape(d, d)  # R[j] = column j
    eps = real(1e-8)
    for j in range(d):
        nrm = real(0)
        for i in range(d):
            nrm = real(nrm + R[j, i] * R[j, i])
        nrm = np.sqrt(nrm)
        if nrm < eps:
            nrm = eps
        R[j] = R[j] / nrm
        if j + 1 < d:
            rest = R[j + 1:]
            dot = np.zeros(d - j - 1, dtype=real)
            for i in range(d):
                dot = dot + R[j, i] * rest[:, i]
            R[j + 1:] = rest - dot[:, None] * R[j][None, :]
    return R.reshape(-1)


def _blocks(state, p, real):
    D = 1 << p
    nb = (len(state) + D - 1) // D
    v = np.zeros(nb * 2 * D, dtype=real)
    v[:2 * len(state)] = np.ascontiguousarray(state).view(real)
    return v.reshape(nb, 2 * D)


def _rotate(M, x):
    """out[:, i] = sum_j M[j d + i] x[:, j], sequential over j"""
    d = x.shape[1]
    Mm = M.reshape(d, d)
    out = np.zeros_like(x)
    for j in range(d):
        out = out + Mm[j][None, :] * x[:, j:j + 1]
    return out


def _range(scale, bits, real):
    lo = real(-3) * scale
    hi = real(3) * scale
    step = (hi - lo) / real(1 << bits)
    return lo, hi, step


def record_dtype(nwords, real):
    return np.dtype([("D", "<u8"), ("BITS", "<i4"), ("init", "u1"), ("seed", "<u8"), ("scale", np.dtype(real).newbyteorder("<")),
                     ("nw", "<u8"), ("w", "<u8", (nwords,))])


def encode(state, p, bits, seed, R=None):
    """the file bytes of `state` (complex64 -> fp32 file, complex128 -> fp64 file)"""
    real = np.float32 if state.dtype == np.complex64 else np.float64
    D, d = 1 << p, 2 << p
    if R is None:
        R = rotation(d, seed, real)
    v = _blocks(state, p, real)
    w = _rotate(R, v)
    s = np.zeros(len(v), dtype=real)
    for j in range(d):
        s = s + w[:, j] * w[:, j]
    scale = np.sqrt(s / real(d) + real(1e-8))
    lo, hi, step = _range(scale, bits, real)
    top = (hi - step)[:, None]
    m = np.where(w < top, w, top)
    c = np.where(lo[:, None] < m, m, lo[:, None])
    with np.errstate(divide="ignore", invalid="ignore"):
        q = ((c - lo[:, None]) / step[:, None])
    q = np.where(np.isfinite(q), q, 0).astype(np.int64)
    q = np.clip(q, 0, (1 << bits) - 1)
    q = np.where((step < real(1e-8))[:, None], 0, q).astype(np.uint64)
    nwords = (d * bits + 63) // 64
    words = np.zeros((len(v), nwords + 1), dtype=np.uint64)
    for j in range(d):
        off = j * bits
        wi, bit = off >> 6, off & 63
        words[:, wi] |= q[:, j] << np.uint64(bit)
        if bit + bits > 64:
            words[:, wi + 1] |= q[:, j] >> np.uint64(64 - bit)
    rec = np.zeros(len(v), dtype=record_dtype(nwords, real))
    rec["D"], rec["BITS"], rec["init"], rec["seed"] = D, bits, 1, seed
    rec["scale"], rec["nw"], rec["w"] = scale, nwords, words[:, :nwords]
    hdr = np.array([len(state), D, len(v)], dtype="<u8")
    return hdr.tobytes() + rec.tobytes()


def parse(data, prec):
    """(capacity, p, bits, records) of a file whose every record is initialized"""
    real = np.float32 if prec == 32 else np.float64
    cap, D, nb = (int(x) for x in np.frombuffer(data[:24], dtype="<u8"))
    bits = int(np.frombuffer(data[32:36], dtype="<i4")[0])
    d = 2 * D
    nwords = (d * bits + 63) // 64
    rec = np.frombuffer(data[24:], dtype=record_dtype(nwords, real))
    assert len(rec) == nb and (rec["D"] == D).all() and (rec["nw"] == nwords).all()
    return cap, D.bit_length() - 1, bits, rec


def decode(data, prec):
    """the amplitudes the file decodes to"""
    real = np.float32 if prec == 32 else np.float64
    cap, p, bits, rec = parse(data, prec)
    d = 2 << p
    scale = np.where(rec["init"] != 0, rec["scale"], real(1)).astype(real)
    lo, hi, step = _range(scale, bits, real)
    words = np.concatenate([rec["w"], np.zeros((len(rec), 1), dtype=np.uint64)], axis=1)
    mask = np.uint64((1 << bits) - 1)
    u = np.zeros((len(rec), d), dtype=real)
    for j in range(d):
        off = j * bits
        wi, bit = off >> 6, off & 63
        q = (words[:, wi] >> np.uint64(bit)) & mask
        if bit + bits > 64:
            q |= (words[:, wi + 1] << np.uint64(64 - bit)) & mask
        u[:, j] = lo + (q.astype(real) + real(0.5)) * step
    out = np.empty_like(u)
    for seed in np.unique(rec["seed"]):
        sel = rec["seed"] == seed
        RT = rotation(d, int(seed), real).reshape(d, d).T.reshape(-1)
        out[sel] = _rotate(RT, u[sel])
    cplx = np.complex64 if prec == 32 else np.complex128
    return out.reshape(-1).view(cplx)[:cap].copy()
