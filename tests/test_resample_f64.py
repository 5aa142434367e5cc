"""The resampler stage against a float64 restatement, at every sample format, resampler and pitch edge.

The restatement below re-derives, in numpy, what core/voice.cpp does to turn a voice's buffer into
its resampled line: LoadResampledSamples (:642-811) chunk by chunk with CalculateBufferSize
(:600-640), LoadBufferStatic / LoadBufferQueue (:500-544, :563-594), the sample decoding of
LoadSamples (fmt_traits.h, the G.711 expansions restated from the standard below) and the
position, loop, queue and state update after the mix (:1119-1232).  It shares no control code
with the CPU oracle or the CUDA kernel.  Sample values are exact float32; the only float64
arithmetic is the filter sum, over the reference's float32 coefficients: the phase tables and
BsincPrepare's scale factor and tap count come from the oracle, whose tables and states
tests/test_oracle_vs_ref.py pins bit for bit against the reference.

What each voice mixes is its line, observed one voice per output row:
  - "dry":     a 4-channel device without post-processing (the register-dry k_mix_voices),
               one-hot dry gains of 1.0, as many devices as the scene needs;
  - "parked":  a 16-channel one (the parking k_mix_voices, the dry bus summed past it), run
               with B200MIX_PANMIX_SIMT=1 and on the tensor cores (80 more playing voices with
               zero gains make the bus big enough for them; the launch counts show they ran);
  - "hrtf":    an HRTF device (the parking kernel with kSiHrtf, as bench.py runs) whose HRIRs are
               a unit impulse at tap 0 on one ear, delay 0, gain 1: each ear is one voice's line;
  - "scale":   4096 HRTF voices with impulse HRIRs of random gains on both ears, summed per ear.
Copy-path and point lines, positions, fractions, flags and buffers_done must match exactly.  The
other resamplers' lines must satisfy, per sample,
        |y - y64| <= (m + 8) * u * sum_j T_j |s_j|,     u = 2^-24,
        T_j = |fil| + |sf*scd| + |pf*phd| + |pf*sf*spd|   (cubic: |fil| + |pf*phd|),
which covers a serial float32 sum and the kernel's four partial sums of FFMA2 products over
pre-combined coefficients.  Linear is a + (b - a)*mu, bounded with the terms |a|, mu|a|, mu|b|.

Without a GPU this holds the CPU oracle to the restatement, and checks that the checker rejects
a restatement that is off by one window sample of 2^-15, one phase row or one tap.  With one
(-m gpu) it holds libb200mix.so to the restatement in every shape, and its positions and states
to the restatement and the oracle exactly.

The scenes include the windows whose history comes from a float format while the span after it
is 16-bit: a float32 / int16 queue whose update ends just past the type boundary, and a float32
static voice re-pointed to an int16 buffer without a reset, both with values above 1.  The 16-bit
window must not be packed from such a history."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from helpers import mixlib
from helpers.mixlib import MixDevice
from pyb200mix import abi

f32 = np.float32
U = 2.0 ** -24
EDGE, PAD = 24, abi.PADDING                      # MaxResamplerEdge, MaxResamplerPadding
RESBUF = abi.LINE + 256 + PAD                    # DeviceBase::mResampleData
SRC_MAX = RESBUF - EDGE
ONE = 1 << 16
PHASES = 32
BSINC = (abi.RS_FAST_BSINC12, abi.RS_BSINC12, abi.RS_FAST_BSINC24, abi.RS_BSINC24,
         abi.RS_FAST_BSINC48, abi.RS_BSINC48)
FULL_BSINC = (abi.RS_BSINC12, abi.RS_BSINC24, abi.RS_BSINC48)
FORMATS = (abi.FMT_U8, abi.FMT_I16, abi.FMT_I32, abi.FMT_F32, abi.FMT_F64, abi.FMT_MULAW, abi.FMT_ALAW)
NP_TYPE = {abi.FMT_U8: np.uint8, abi.FMT_I16: np.int16, abi.FMT_I32: np.int32, abi.FMT_F32: np.float32,
           abi.FMT_F64: np.float64, abi.FMT_MULAW: np.uint8, abi.FMT_ALAW: np.uint8}
SIZES = [1024, 1, 517, 2, 65, 3, 1023, 4, 129, 63, 128, 64, 127]
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


# ---- G.711 (ITU-T G.711 expansion, scaled to 16 bits) ----------------------------------------
def _mulaw():
    out = np.zeros(256, np.int32)
    for code in range(256):
        u = ~code & 0xff
        seg, q = (u >> 4) & 7, u & 15
        mag = (((2 * q + 33) << seg) - 33) * 4          # 14-bit magnitude, times 4
        out[code] = -mag if u & 0x80 else mag
    return out


def _alaw():
    out = np.zeros(256, np.int32)
    for code in range(256):
        a = code ^ 0x55
        seg, q = (a >> 4) & 7, a & 15
        mag = (2 * q + 1) if seg == 0 else ((2 * q + 33) << (seg - 1))
        mag *= 8                                        # 13-bit magnitude, times 8
        out[code] = mag if a & 0x80 else -mag
    return out


MULAW, ALAW = _mulaw(), _alaw()


def decode(fmt, raw):
    """LoadSamples' conversion to float32 (fmt_traits.h): exact, but i32 and f64 round once."""
    if fmt == abi.FMT_U8:
        return (raw.astype(f32) - f32(128.0)) * f32(1.0 / 128.0)
    if fmt == abi.FMT_I16:
        return raw.astype(f32) * f32(2.0 ** -15)
    if fmt == abi.FMT_I32:
        return raw.astype(f32) * f32(2.0 ** -31)
    if fmt in (abi.FMT_F32, abi.FMT_F64):
        return raw.astype(f32)
    table = MULAW if fmt == abi.FMT_MULAW else ALAW
    return table[raw].astype(f32) * f32(2.0 ** -15)


class Buf:
    def __init__(self, fmt, raw):
        self.fmt, self.raw = fmt, np.ascontiguousarray(raw)         # raw: [frames][channels]
        self.frames, self.channels = raw.shape
        self.dec = decode(fmt, self.raw)

    def samples(self, chan, start, count):
        ch = chan if chan < self.channels else 0                       # a channel it lacks: 0
        return self.dec[start:start + count, ch]


# ---- tables --------------------------------------------------------------------------------
_TABLES = {}


def _oracle():
    lib = mixlib.oracle().lib
    lib.oracle_get_resampler_table.restype = C.c_int64
    lib.oracle_get_resampler_table.argtypes = [C.c_uint32, C.c_void_p, C.c_size_t]
    lib.oracle_get_bsinc_state.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_float),
                                           C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                           C.POINTER(C.c_uint32)]
    return lib


def table(which):
    if which not in _TABLES:
        lib = _oracle()
        n = lib.oracle_get_resampler_table(which, None, 0)
        t = np.zeros(n, f32)
        lib.oracle_get_resampler_table(which, t.ctypes.data, n)
        _TABLES[which] = t
    return _TABLES[which]


def bsinc_state(which, inc):
    """(sf, m, l, offset) of BsincPrepare."""
    key = (which, inc)
    if key not in _TABLES:
        o = (C.c_float(), C.c_uint32(), C.c_uint32(), C.c_uint32())
        assert _oracle().oracle_get_bsinc_state(which, inc, *[C.byref(x) for x in o]) == 0
        _TABLES[key] = (f32(o[0].value), o[1].value, o[2].value, o[3].value)
    return _TABLES[key]


def scale_boundaries(which):
    """The increments at which BsincPrepare moves to the next filter scale."""
    key = ("bounds", which)
    if key not in _TABLES:
        incs = np.arange(ONE + 1, (10 << 16) + 1, 1024)
        offs = [bsinc_state(which, int(i))[3] for i in incs]
        out = []
        for a in range(len(incs) - 1):
            if offs[a] == offs[a + 1]:
                continue
            lo, hi = int(incs[a]), int(incs[a + 1])           # offset(lo) != offset(hi)
            while hi - lo > 1:
                mid = (lo + hi) // 2
                if bsinc_state(which, mid)[3] == offs[a]:
                    lo = mid
                else:
                    hi = mid
            out.append(hi)
        _TABLES[key] = out
    return _TABLES[key]


def buffer_size(frac, inc, remaining):
    """CalculateBufferSize: (dst, src) of the next chunk."""
    ext = 1 if inc <= ONE else 0
    src = (((remaining - ext) * inc + frac) >> 16) + ext + EDGE
    if src <= SRC_MAX:
        return remaining, src
    dst = (((SRC_MAX - EDGE) << 16) - frac) // inc
    if dst < remaining:
        return dst & ~3, SRC_MAX
    return remaining, SRC_MAX


def add_sat(a, b):
    return max(INT32_MIN, min(INT32_MAX, a + b))


# ---- the restatement ----------------------------------------------------------------------
def resample(rs, inc, frac, rd, dstn, perturb=None):
    """One chunk through resampler rs: (line in float64, per-sample bound).  perturb: None,
    "phase" (output 0 uses phase row pi+1) or "tap" (every output reads one tap later)."""
    fp = np.arange(dstn, dtype=np.int64) * inc + frac
    pos, fr = fp >> 16, fp & 0xffff
    if rs == abi.RS_POINT:
        return rd[EDGE + pos].astype(np.float64), np.zeros(dstn)
    if rs == abi.RS_LINEAR:
        a = rd[EDGE + pos].astype(np.float64)
        b = rd[EDGE + pos + 1].astype(np.float64)
        mu = fr / 65536.0
        return a + mu * (b - a), 10.0 * U * (np.abs(a) + mu * (np.abs(a) + np.abs(b)))
    pi = fr >> 11
    pf = (fr & 2047) / 2048.0
    if rs in (abi.RS_SPLINE, abi.RS_GAUSSIAN):
        tab = table(rs).reshape(PHASES, 8).astype(np.float64)
        m, base, sf = 4, EDGE - 1, 0.0
        F, D = tab[:, :4], tab[:, 4:]
        SC = SP = np.zeros_like(F)
    else:
        sf, m, l, off = bsinc_state(rs, inc)
        sf = float(sf) if (inc > ONE and rs in FULL_BSINC) else 0.0
        t = table(rs)[off:].astype(np.float64)
        rows = t[:2 * PHASES * m].reshape(PHASES, 2, m)
        F, D = rows[:, 0], rows[:, 1]
        if sf:
            rows = t[2 * PHASES * m:4 * PHASES * m].reshape(PHASES, 2, m)
            SC, SP = rows[:, 0], rows[:, 1]
        else:
            SC = SP = np.zeros_like(F)
        base = EDGE - l
    if perturb == "phase":
        pi = pi.copy()
        pi[0] = (pi[0] + 1) % PHASES
    if perturb == "tap":
        base += 1
    s = rd[base + pos[:, None] + np.arange(m)[None, :]].astype(np.float64)
    pfc = pf[:, None]
    c = F[pi] + sf * SC[pi] + pfc * (D[pi] + sf * SP[pi])
    T = np.abs(F[pi]) + np.abs(sf * SC[pi]) + np.abs(pfc * D[pi]) + np.abs(pfc * sf * SP[pi])
    return (c * s).sum(axis=1), (m + 8) * U * (T * np.abs(s)).sum(axis=1)


class Voice:
    """One voice's mixing state (core/voice.h), as the update parameters set it."""

    def __init__(self, bufs):
        self.bufs = bufs
        self.state = 0
        self.prev = np.zeros(PAD, f32)
        self.queue, self.qloop, self.qhead = [], None, 0
        self.have_buffer = False
        self.pos = self.frac = self.done = 0
        self.faded = False          # mixed while stopping since: its gains ramp up again

    def set_queue(self, items, loop):
        self.queue, self.qloop, self.qhead = list(items), (None if loop == abi.NO_LOOP else loop), 0
        self.have_buffer = len(items) > 0

    def update(self, p):
        if p.flags & abi.VF_RESET:
            self.prev = np.zeros(PAD, f32)
            self.pos, self.frac, self.have_buffer, self.qhead = p.position, p.position_frac, True, 0
            self.faded = False
        if p.flags & abi.VF_STOPPED:
            self.state = 0
        elif p.flags & abi.VF_STOPPING:
            self.state = 2
        elif p.flags & abi.VF_PLAYING:
            self.state = 1
        self.static = bool(p.flags & abi.VF_STATIC)
        self.looping = bool(p.flags & abi.VF_LOOPING)
        self.chan = (p.flags >> 16) & 0xff
        self.buf = p.buffer
        if p.buffer == 0xFFFFFFFF:
            self.have_buffer = False
        self.ls, self.le, self.step, self.rs = p.loop_start, p.loop_end, p.step, p.resampler

    def _next(self, item):
        return item + 1 if item + 1 < len(self.queue) else self.qloop

    def _static(self, looping, pos, dst):
        b = self.bufs[self.buf]
        if not looping:
            last = f32(0.0)
            if b.frames > pos:
                r = min(len(dst), b.frames - pos)
                dst[:r] = b.samples(self.chan, pos, r)
                last = dst[r - 1]
                dst = dst[r:]
            dst[:] = last
            return
        ls, le = self.ls, self.le
        ip = pos if pos < le else (pos - ls) % (le - ls) + ls
        r = min(len(dst), le - ip)
        dst[:r] = b.samples(self.chan, ip, r)
        rest = len(dst) - r
        if rest:
            loop = b.samples(self.chan, ls, le - ls)
            dst[r:] = loop[np.arange(rest) % (le - ls)]

    def _queue(self, pos, dst):
        last, item, i = f32(0.0), self.qhead, 0
        while item is not None and i < len(dst):
            b = self.bufs[self.queue[item]]
            if pos >= b.frames:
                pos -= b.frames
                item = self._next(item)
                continue
            r = min(len(dst) - i, b.frames - pos)
            dst[i:i + r] = b.samples(self.chan, pos, r)
            last = dst[i + r - 1]
            i += r
            if i == len(dst):
                break
            pos, item = 0, self._next(item)
        dst[i:] = last

    def mix(self, n, perturb=None):
        """Voice::mix for n samples: (line, bound, observed) or None.  The line is observed (at
        gain 1) when the voice plays, and did not fade out while stopping since its reset."""
        if self.state not in (1, 2):
            return None
        inc = self.step
        if inc < 1:
            if self.state == 2:
                self.state = 0
            return None
        looping = self.looping
        if self.static and looping and self.have_buffer and self.pos >= self.le:
            looping = False                                    # core/voice.cpp:1015-1019
        playing = self.state == 1
        y, tol = np.zeros(n), np.zeros(n)
        rd = np.zeros(RESBUF, f32)
        rd[:PAD] = self.prev
        ipos, frac, loaded, first = self.pos, self.frac, 0, True
        while loaded < n:
            dstn, srcn = buffer_size(frac, inc, n - loaded)
            delay = 0
            if ipos < 0:
                delay = -ipos
                if delay >= srcn:                              # silent: no history, no slide
                    rd[EDGE:EDGE + srcn] = 0.0
                    loaded += dstn
                    if loaded < n:
                        frac += dstn * inc
                        ipos, frac = add_sat(ipos, frac >> 16), frac & 0xffff
                    continue
                rd[EDGE:EDGE + delay] = 0.0
            if not self.have_buffer:
                # ended: hold the first of the samples nearest 0 (core/voice.cpp:704-719)
                avail, tofill = min(srcn, EDGE), max(srcn, EDGE)
                best = int(np.argmin(np.abs(rd[EDGE:EDGE + avail])))
                rd[EDGE + best + 1:EDGE + tofill] = rd[EDGE + best]
            elif self.static:
                self._static(looping, max(ipos, 0), rd[EDGE + delay:EDGE + srcn])
            else:
                self._queue(max(ipos, 0), rd[EDGE + delay:EDGE + srcn])
            p = perturb if first else None
            if inc == ONE and frac == 0:
                if p == "sample":
                    rd[EDGE] += f32(2.0 ** -15)
                y[loaded:loaded + dstn] = rd[EDGE:EDGE + dstn]
            else:
                if p == "sample":
                    # the sample output 0 weighs most
                    y0, _ = resample(self.rs, inc, frac, rd, 1)
                    best, gain = EDGE, -1.0
                    for k in range(max(0, EDGE - 24), EDGE + 26):
                        r2 = rd.copy()
                        r2[k] += f32(1.0)
                        d = abs(float(resample(self.rs, inc, frac, r2, 1)[0][0] - y0[0]))
                        if d > gain:
                            best, gain = k, d
                    rd[best] += f32(2.0 ** -15)
                yy, tt = resample(self.rs, inc, frac, rd, dstn, perturb=p if p != "sample" else None)
                y[loaded:loaded + dstn], tol[loaded:loaded + dstn] = yy, tt
            first = False
            if playing and loaded < n <= loaded + dstn:
                off = ((n - loaded) * inc + frac) >> 16
                self.prev = rd[off:off + PAD].copy()
            loaded += dstn
            if loaded < n:
                frac += dstn * inc
                off = frac >> 16
                frac &= 0xffff
                ipos = ipos + off if ipos < 0 else add_sat(ipos, off)
                rd[:PAD] = rd[off:off + PAD].copy()
        settled = playing and not self.faded
        self.faded = not playing
        if self.state == 2:
            self.state = 0
            return y, tol, False
        # positions, loops, queue and state (core/voice.cpp:1125-1232)
        self.done = 0
        frac = self.frac + inc * n
        pos = add_sat(self.pos, frac >> 16)
        self.frac = frac & 0xffff
        if self.have_buffer and pos > 0:
            if not self.static:
                item = self.qhead
                while item is not None:
                    ln = self.bufs[self.queue[item]].frames
                    if ln > pos:
                        break
                    pos -= ln
                    self.done += 1
                    item = self._next(item)
                if item is None:
                    self.have_buffer = False
                else:
                    self.qhead = item
            elif looping:
                if pos >= self.le:
                    pos = (pos - self.ls) % (self.le - self.ls) + self.ls
            elif pos >= self.bufs[self.buf].frames:
                self.have_buffer = False
        self.pos = pos
        if not self.have_buffer:
            self.state = 2
        return y, tol, settled

    def result(self):
        flags = abi.VF_PLAYING if self.state == 1 else abi.VF_STOPPING if self.state == 2 else abi.VF_STOPPED
        return (self.pos, self.frac, flags, self.done)


# ---- scenes --------------------------------------------------------------------------------
def _values(rng, fmt, frames, chans, loud):
    shape = (frames, chans)
    if fmt == abi.FMT_U8:
        raw = rng.integers(0, 256, shape).astype(np.uint8)
        ext = (0, 255)
    elif fmt == abi.FMT_I16:
        raw = rng.integers(-32768, 32768, shape).astype(np.int16)
        ext = (-32768, 32767)
    elif fmt == abi.FMT_I32:
        raw = rng.integers(INT32_MIN, INT32_MAX, shape, endpoint=True).astype(np.int32)
        ext = (INT32_MIN, INT32_MAX)
    elif fmt in (abi.FMT_F32, abi.FMT_F64):
        x = rng.uniform(-1.0, 1.0, shape) * (3.0 if loud else 1.0)
        x = np.where(np.abs(x) < 1e-6, 0.5, x)             # nothing near the denormal range
        raw = x.astype(NP_TYPE[fmt])
        ext = (-1.0, 1.0, 3.5) if loud else (-1.0, 1.0)
    else:
        raw = rng.integers(0, 256, shape).astype(np.uint8)
        ext = (0x00, 0x80, 0x7f, 0xff)
    k = rng.integers(0, frames * chans, min(6, frames * chans))
    flat = raw.reshape(-1)
    for i, e in zip(k, np.resize(np.array(ext), len(k))):
        flat[i] = e
    return Buf(fmt, raw)


KINDS = ("loop_big", "loop1", "loop2", "loop3", "loop_lt_m", "loop_lt_win", "oneshot_end", "neg",
         "neg_srcn", "past_loop_end", "buf1", "buf2", "buf_short", "queue_1frame", "queue_loop_mid",
         "queue_runout", "no_buffer")
FRACS = (0, 1, 2047, 2048, 65535)


def _steps(rs, k):
    """The step axis: every edge, with bsinc scale boundaries from the voice's own table."""
    bt = rs if rs in BSINC else abi.RS_BSINC24
    bounds = scale_boundaries(bt)
    b = bounds[(k // 13) % len(bounds)] - (k // 7) % 2
    return [1, 0x8000, 65535, ("copy", ONE), ONE, 65537, "two_chunk", b, 2 << 16, 216268, 10 << 16,
            int(1.25 * ONE) + 3, 0x18000]


def _resolve(st, frac):
    """(step, fraction) of an entry of _steps."""
    if st == ("copy", ONE):
        return ONE, 0                                          # the copy path
    if st == ONE and frac == 0:
        return ONE, 2047
    if st == "two_chunk":                                      # the first step that splits 1024
        return -(-(1281 * ONE - frac) // 1023), frac
    return st, frac


class Spec:
    """What one voice is given: buffers, initial parameters, queue, changes per update."""

    def __init__(self):
        self.bufs, self.queue, self.events = [], None, {}


def _params(flags, buf, rs, pos, frac, ls, le, step):
    p = abi.VoiceParams()
    p.flags, p.buffer, p.resampler = flags, buf, rs
    p.position, p.position_frac, p.loop_start, p.loop_end, p.step = pos, frac, ls, le, step
    p.hrtf_gain = 1.0
    for s in range(abi.MAX_SENDS):
        p.send_slot[s] = abi.NO_SLOT
    return p


def scene(nv, seed, sizes=SIZES):
    """nv voices; voice k takes one value along each axis (cycled, so that every format x
    resampler pair appears within 70 voices)."""
    rng = np.random.default_rng(seed)
    specs = []
    n0 = sizes[0]
    for k in range(nv):
        sp = Spec()
        fmt = FORMATS[k % 7]
        rs = (k // 7) % 10
        chans = (1, 2, 4)[k % 3]
        chan = (k // 3) % (chans + 1)                          # chans: a channel it lacks
        kind = KINDS[k % len(KINDS)]
        steps = _steps(rs, k)
        st, frac = _resolve(steps[k % len(steps)], FRACS[(k // 5) % 5])
        loud = k % 2 == 0
        frames = int(rng.integers(3000, 7000))
        flags = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_RESET | abi.vf_channel(chan)
        ls, le, pos = 0, frames, int(rng.integers(0, frames))
        lead = k % 8
        if kind.startswith("loop"):
            flags |= abi.VF_LOOPING
            size = {"loop_big": frames // 2, "loop1": 1, "loop2": 2, "loop3": 3,
                    "loop_lt_m": int(rng.integers(4, 12)), "loop_lt_win": int(rng.integers(40, 700))}[kind]
            ls = 8 * int(rng.integers(1, (frames - size) // 8 - 1)) + lead
            le = ls + size
            pos = int(rng.integers(0, le))
        elif kind == "oneshot_end":
            pos = frames - 1
        elif kind == "neg":
            srcn = buffer_size(frac, st, n0)[1]
            pos = -[srcn // 2, srcn + 7, 5 * srcn + 100, 1][(k // 17) % 4]
            if k % 2:
                flags |= abi.VF_LOOPING
        elif kind == "neg_srcn":
            pos = -buffer_size(frac, st, n0)[1]
        elif kind == "past_loop_end":
            flags |= abi.VF_LOOPING
            ls = 8 * int(rng.integers(1, 100)) + lead
            le = ls + int(rng.integers(50, 2000))
            pos = le + (0 if (k // 17) % 2 == 0 else int(rng.integers(1, 300)))
        elif kind in ("buf1", "buf2", "buf_short"):
            frames = {"buf1": 1, "buf2": 2, "buf_short": int(rng.integers(3, 60))}[kind]
            pos, le = 0, frames
            if k % 2:
                flags |= abi.VF_LOOPING
        sp.bufs.append(_values(rng, fmt, frames, chans, loud))
        if kind.startswith("queue"):
            flags &= ~abi.VF_STATIC
            lens = {"queue_1frame": [1, 1, 40, 1, 3000, 1],
                    "queue_loop_mid": [int(x) for x in rng.integers(5, 300, 6)],
                    "queue_runout": [700, 30, 400]}[kind]
            sp.bufs = [_values(rng, fmt, ln, chans, loud) for ln in lens]
            loop = 2 if kind == "queue_loop_mid" else abi.NO_LOOP
            if kind == "queue_1frame":
                loop = 0
            sp.queue = (list(range(len(lens))), loop)
            pos = int(rng.integers(0, 20))
            if kind == "queue_runout":
                pos = 1100 - int(st * 1000 // ONE) % 900       # runs out within a few updates
        if kind == "no_buffer":
            sp.events[3] = [("nobuffer",)]
        sp.p0 = _params(flags, 0, rs, pos, frac, ls, le, st)
        # mid-run: stops, and step changes without a reset
        if k % 11 == 4:
            sp.events.setdefault(5 + k % 4, []).append(("stop",))
        if k % 6 == 1:
            sp.events.setdefault(2 + k % 5, []).append(("step", _resolve(steps[(k + 5) % len(steps)], 1)[0]))
        specs.append(sp)
    return specs


def defect_scene(seed, sizes):
    """Windows whose history is float32 above full scale while their span is int16: a mixed
    float32 / int16 queue whose first update ends 1..23 samples past the type boundary, and a
    float32 static voice re-pointed to int16 buffers (mono through the bulk copy, stereo and u8
    through the gather) without a reset.  All bsinc, packed-window steps."""
    rng = np.random.default_rng(seed)
    specs = []
    n0 = sizes[0]
    for k in range(48):
        sp = Spec()
        rs = BSINC[k % 6]
        step = (0x8000, 0xC000, 65537, 0x14000)[(k // 6) % 4]
        frac = FRACS[1 + k % 4]
        # the float buffer outlasts update 0: a re-pointed voice still plays when it is re-pointed
        f0 = 600 + 8 * k + ((n0 * step + frac) >> 16)
        loudf = _values(rng, abi.FMT_F32, f0, 1, True)
        loudf.raw[-3:] = np.array([[1.0], [-3.25], [1.0]], f32)
        loudf.dec = decode(abi.FMT_F32, loudf.raw)
        if k < 24:
            # the queue: update 0 consumes floor((n0*step + frac) / 65536) samples
            d = 1 + k % 23
            pos = f0 + d - ((n0 * step + frac) >> 16)
            sp.bufs = [loudf, _values(rng, abi.FMT_I16, 4000, 1, False)]
            sp.queue = ([0, 1], abi.NO_LOOP)
            flags = abi.VF_PLAYING | abi.VF_RESET
            sp.p0 = _params(flags, 0, rs, pos, frac, 0, 0, step)
        else:
            fmt, chans = ((abi.FMT_I16, 1), (abi.FMT_I16, 2), (abi.FMT_U8, 1))[k % 3]
            sp.bufs = [loudf, _values(rng, fmt, 4000, chans, False)]
            flags = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_RESET
            sp.p0 = _params(flags, 0, rs, 20 + k % 8, frac, 0, f0, step)
            sp.events[1] = [("repoint", 1)]
        specs.append(sp)
    return specs


def boundary_scene(seed, sizes):
    """Every bsinc and fast bsinc resampler at every scale boundary of its table: the first step
    BsincPrepare gives the next scale, and the step below it.  Formats and channel counts cycle."""
    rng = np.random.default_rng(seed)
    specs = []
    i = 0
    for rs in BSINC:
        for b in scale_boundaries(rs):
            for step in (b, b - 1):
                sp = Spec()
                fmt, chans = FORMATS[i % 7], (1, 2, 4)[i % 3]
                sp.bufs = [_values(rng, fmt, 3000, chans, i % 2 == 0)]
                flags = (abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING | abi.VF_RESET
                         | abi.vf_channel(i % (chans + 1)))
                ls = 8 * int(rng.integers(1, 40)) + i % 8
                sp.p0 = _params(flags, 0, rs, int(rng.integers(0, 3000)), FRACS[i % 5], ls, 3000, step)
                specs.append(sp)
                i += 1
    return specs


# ---- running a scene ---------------------------------------------------------------------
def _changed(p, ev):
    q = abi.VoiceParams.from_buffer_copy(bytes(p))
    q.flags &= ~abi.VF_RESET
    for e in ev:
        if e[0] == "stop":
            q.flags = (q.flags & ~abi.VF_PLAYING) | abi.VF_STOPPING
        elif e[0] == "step":
            q.step = e[1]
        elif e[0] == "repoint":
            q.buffer = e[1]
        elif e[0] == "nobuffer":
            q.buffer = 0xFFFFFFFF
    return q


def restate(specs, sizes, perturb=None):
    """[(lines [nv][n], bounds, checked [nv], results [nv])] per update."""
    vs = [Voice(sp.bufs) for sp in specs]
    params = [sp.p0 for sp in specs]
    for v, sp in zip(vs, specs):
        if sp.queue:
            v.set_queue(*sp.queue)
        v.update(sp.p0)
    out = []
    for u, n in enumerate(sizes):
        for k, sp in enumerate(specs):
            if u in sp.events:
                params[k] = _changed(params[k], sp.events[u])
                vs[k].update(params[k])
        lines, bounds, checked = np.zeros((len(vs), n)), np.zeros((len(vs), n)), np.zeros(len(vs), bool)
        for k, v in enumerate(vs):
            v.done = 0
            r = v.mix(n, perturb)
            if r is not None:
                lines[k], bounds[k], checked[k] = r
        out.append((lines, bounds, checked, [v.result() for v in vs]))
    return out


SHAPES = {"dry": 4, "parked": 16, "hrtf": 2}
# playing voices with zero dry gains beside a parked device's 16: the dry bus then has more than 64
# entries (two chunks), which is when a full update's pan-mix runs on the tensor cores
PARK_PAD = 80


def _desc(shape, nv):
    d = abi.DeviceDesc()
    d.struct_size = C.sizeof(abi.DeviceDesc)
    d.cuda_device, d.sample_rate = -1, 48000
    d.max_voices, d.max_buffers, d.max_slots = nv, 8 * nv, 0
    if shape in ("hrtf", "scale"):
        d.dry_channels, d.real_channels, d.ir_size, d.post_process = 4, 2, 8, abi.POST_HRTF
    else:
        d.dry_channels = d.real_channels = SHAPES[shape]
        d.post_process = abi.POST_NONE
    d.real_left, d.real_right = 0, 1
    return d


def play(lib, specs, sizes, shape="dry", ir=8, gains=None, launches=None):
    """Runs the scene on one implementation: [(rows [nv][n] float32, results)] per update.  Each
    device of the shape holds SHAPES[shape] voices and gives one row per voice; "scale" is one
    device whose two rows are the ears' gain-weighted sums.  A "parked" device also plays
    PARK_PAD silent voices.  launches: a list that gets each product device's launch count."""
    nv = len(specs)
    per = nv if shape == "scale" else SHAPES[shape]
    out = [(np.zeros((2 if shape == "scale" else nv, n), f32), [None] * nv) for n in sizes]
    for d0 in range(0, nv, per):
        ks = list(range(d0, min(d0 + per, nv)))
        pad = PARK_PAD if shape == "parked" else 0
        desc = _desc(shape, len(ks) + pad)
        if shape in ("hrtf", "scale"):
            desc.ir_size = ir
        dev = MixDevice(lib, desc)
        if shape in ("hrtf", "scale"):
            dec = np.zeros((4, 8, 2), f32)
            dev.set_hrtf_decoder(dec, np.ones(4, f32), np.zeros(4, f32))
        coeffs = np.zeros((len(ks), ir, 2), f32)
        dry = np.zeros((len(ks) + pad, desc.dry_channels), f32)
        for s, k in enumerate(ks):
            if shape == "scale":
                coeffs[s, 0] = gains[k]
            elif shape == "hrtf":
                coeffs[s, 0, s] = 1.0
            else:
                dry[s, s] = 1.0
            for j, b in enumerate(specs[k].bufs):
                dev.buffer_data(8 * s + j, b.fmt, b.raw, channels=b.channels)
            if specs[k].queue:
                items, loop = specs[k].queue
                dev.voice_queue(s, [8 * s + j for j in items], loop)
        params = []
        for s, k in enumerate(ks):
            p = abi.VoiceParams.from_buffer_copy(bytes(specs[k].p0))
            p.voice, p.buffer = s, 8 * s + p.buffer
            if shape in ("hrtf", "scale"):
                p.flags |= abi.VF_HRTF
            params.append(p)
        if pad:
            dev.buffer_data(8 * len(ks), abi.FMT_I16, (np.arange(1024) * 37 % 2001 - 1000).astype(np.int16))
        for s in range(len(ks), len(ks) + pad):
            params.append(_params(abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING | abi.VF_RESET,
                                  8 * len(ks), abi.RS_LINEAR, s, 0, 0, 1024, 0x11000))
            params[-1].voice = s
        dev.voices_update(params, coeffs if shape in ("hrtf", "scale") else None, dry, None)
        for u, n in enumerate(sizes):
            upd = []
            for s, k in enumerate(ks):
                if u in specs[k].events:
                    q = _changed(params[s], specs[k].events[u])
                    if q.buffer != 0xFFFFFFFF and any(e[0] == "repoint" for e in specs[k].events[u]):
                        q.buffer = 8 * s + q.buffer
                    params[s] = q
                    upd.append(q)
            if upd:
                dev.voices_update(upd, None, dry[[p.voice for p in upd]], None)
            if shape in ("hrtf", "scale"):
                rows, res = dev.render(n, want_results=True)
            else:
                res = dev.render(n, want_results=True)[1]
                rows = dev.dry()[:, :n]
            if shape == "scale":
                out[u][0][:] = rows
            else:
                out[u][0][ks] = rows[:len(ks)]
            for s, k in enumerate(ks):
                r = res[s]
                out[u][1][k] = (r.position, r.position_frac, r.flags, r.buffers_done)
        if launches is not None:
            fn = lib.lib.b200mix_launch_count
            fn.restype, fn.argtypes = C.c_uint64, [C.c_void_p]
            launches.append(int(fn(dev.h)))
        dev.close()
    return out


def check(got, ref, what, extra=None, sizes=SIZES):
    """Failure messages: rows outside their bounds, results that differ.  extra(u, lines) adds
    a shape's own term to the bound."""
    bad = []
    for u, ((rows, res), (lines, bounds, checked, rres)) in enumerate(zip(got, ref)):
        tol = bounds + (extra(u, lines) if extra else 0.0)
        err = np.abs(rows.astype(np.float64) - lines)
        for k in np.nonzero(checked)[0]:
            if (err[k] > tol[k]).any():
                i = int(np.argmax(err[k] - tol[k]))
                bad.append(f"{what} update {u} (n {sizes[u]}) voice {k}: {int((err[k] > tol[k]).sum())} "
                           f"samples outside the bound, at {i}: got {rows[k, i]!r} want {lines[k, i]!r} "
                           f"bound {tol[k, i]:.3e}")
        for k, want in enumerate(rres):
            if res[k] != want:
                bad.append(f"{what} update {u} voice {k}: result {res[k]} != {want}")
    return bad


def _assert_ok(bad):
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:25])


SCENES = [(170, 11, SIZES), (170, 12, SIZES[::-1]), (170, 13, SIZES[5:] + SIZES[:5])]
DEFECT = [(21, [1024, 1024, 517, 64]), (22, [517, 1023, 3, 1024]), (23, [127, 1024, 65, 129])]


def _silent_guard(ref):
    assert max(float(np.abs(lines).max()) for lines, _, _, _ in ref) > 0.1, "the run is silent"


# ---- CPU half -----------------------------------------------------------------------------
@pytest.mark.parametrize("nv,seed,sizes", SCENES)
def test_oracle_vs_float64(nv, seed, sizes):
    specs = scene(nv, seed, sizes)
    ref = restate(specs, sizes)
    _silent_guard(ref)
    _assert_ok(check(play(mixlib.oracle(), specs, sizes), ref, f"oracle seed {seed}", sizes=sizes))


@pytest.mark.parametrize("seed,sizes", DEFECT)
def test_oracle_vs_float64_float_history(seed, sizes):
    specs = defect_scene(seed, sizes)
    ref = restate(specs, sizes)
    _silent_guard(ref)
    _assert_ok(check(play(mixlib.oracle(), specs, sizes), ref, f"oracle seed {seed}", sizes=sizes))


def test_oracle_vs_float64_scale_boundaries():
    sizes = [1024, 517, 63, 1024]
    specs = boundary_scene(41, sizes)
    ref = restate(specs, sizes)
    _silent_guard(ref)
    _assert_ok(check(play(mixlib.oracle(), specs, sizes), ref, "oracle boundaries", sizes=sizes))


@pytest.mark.parametrize("perturb", ["sample", "phase", "tap"])
def test_checker_rejects_perturbed_restatement(perturb):
    """The bound is tight enough to see one window sample moved by 2^-15, one output on the
    next phase row, or every tap one sample late."""
    nv, seed, sizes = SCENES[0]
    specs = scene(nv, seed, sizes)
    got = play(mixlib.oracle(), specs, sizes)
    assert not check(got, restate(specs, sizes), "oracle", sizes=sizes)
    bad = check(got, restate(scene(nv, seed, sizes), sizes, perturb=perturb), perturb, sizes=sizes)
    voices = {m.split(" voice ")[1].split(":")[0] for m in bad}
    # caught on many voices, not one: "phase" and "tap" leave point, linear and copy lines alone
    assert len(voices) >= (60 if perturb == "sample" else 40), f"{perturb}: only {len(voices)} voices rejected"


# ---- GPU half -----------------------------------------------------------------------------
@contextlib.contextmanager
def _env(name, value):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


def _results_vs_oracle(got, ora, what):
    bad = []
    for u, ((_, res), (_, rres)) in enumerate(zip(got, ora)):
        for k, (a, b) in enumerate(zip(res, rres)):
            if a != b:
                bad.append(f"{what} update {u} voice {k}: {a} != oracle {b}")
    return bad


def _tc_term(u, lines, sizes):
    # 3xTF32 tensor-core pan-mix of full updates: tests/test_gpu_panmix.py's
    # (5*2^-22 + 3*nkb*2^-23) * sum |g x|, where sum |g x| is the row's one voice and a chunk holds
    # at most half of the (at most 16 + PARK_PAD) entries, nkb = its K blocks of 8
    if sizes[u] != abi.LINE:
        return 0.0
    nkb = -(-(-(-(16 + PARK_PAD) // 2)) // 8)
    return (5.0 * 2.0 ** -22 + 3.0 * nkb * 2.0 ** -23) * np.abs(lines)


def _gpu_run(specs, sizes, what):
    ref = restate(specs, sizes)
    _silent_guard(ref)
    ora = play(mixlib.oracle(), specs, sizes)
    bad = []
    got = play(mixlib.product(), specs, sizes, "dry")
    bad += check(got, ref, f"{what} dry", sizes=sizes) + _results_vs_oracle(got, ora, f"{what} dry")
    simt, tc = [], []
    with _env("B200MIX_PANMIX_SIMT", "1"):
        got = play(mixlib.product(), specs, sizes, "parked", launches=simt)
    bad += check(got, ref, f"{what} parked simt", sizes=sizes)
    got = play(mixlib.product(), specs, sizes, "parked", launches=tc)
    bad += check(got, ref, f"{what} parked tc", extra=lambda u, ln: _tc_term(u, ln, sizes), sizes=sizes)
    # k_panmix_tc is the one launch the SIMT switch removes: once per full update on every device
    full = sum(n == abi.LINE for n in sizes)
    if [a - b for a, b in zip(tc, simt)] != [full] * len(tc):
        bad.append(f"{what} parked: tensor-core launches {[a - b for a, b in zip(tc, simt)]}, "
                   f"want {full} per device")
    for ir in (8, 128):
        # the 64-sample blend after the first update: x*old_step*(c-i) + x*new_step*i
        got = play(mixlib.product(), specs, sizes, "hrtf", ir=ir)
        bad += check(got, ref, f"{what} hrtf ir {ir}", extra=lambda u, ln: 4.0 * U * np.abs(ln), sizes=sizes)
    _assert_ok(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("nv,seed,sizes", SCENES)
def test_kernel_vs_float64(nv, seed, sizes):
    _gpu_run(scene(nv, seed, sizes), sizes, f"seed {seed}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed,sizes", DEFECT)
def test_kernel_vs_float64_float_history(seed, sizes):
    _gpu_run(defect_scene(seed, sizes), sizes, f"seed {seed}")


@pytest.mark.gpu
def test_kernel_vs_float64_scale_boundaries():
    sizes = [1024, 517, 63, 1024]
    _gpu_run(boundary_scene(41, sizes), sizes, "boundaries")


@pytest.mark.gpu
def test_kernel_vs_float64_at_scale():
    """4096 HRTF voices (bench config 2's count) summed per ear through impulse HRIRs of random
    gains: |out - sum g y64| <= sum |g| bound + (V + 2) u sum |g y64|."""
    sizes = [1024, 517, 1024, 64, 1024]
    nv = 4096
    specs = scene(nv, 31, sizes)
    gains = np.random.default_rng(5).uniform(-1.0, 1.0, (nv, 2)).astype(f32) / f32(64.0)
    ref = restate(specs, sizes)
    _silent_guard(ref)
    for u, (_, _, checked, _) in enumerate(ref):
        assert checked.sum() >= nv // 2, f"update {u}: only {int(checked.sum())} voices observed"
    got = play(mixlib.product(), specs, sizes, "scale", ir=8, gains=gains)
    ora = play(mixlib.oracle(), specs, sizes, "scale", ir=8, gains=gains)
    bad = _results_vs_oracle(got, ora, "scale")
    for u, ((rows, res), (lines, bounds, checked, rres)) in enumerate(zip(got, ref)):
        for k, want in enumerate(rres):
            if res[k] != want:
                bad.append(f"scale update {u} voice {k}: result {res[k]} != {want}")
        # the lines of stopping voices fade with their gain: none of those are summed here
        live = checked.copy()
        for e in range(2):
            g = gains[:, e].astype(np.float64)[:, None]
            want = (g * lines)[live].sum(axis=0)
            tol = ((np.abs(g) * (bounds + 4.0 * U * np.abs(lines)))[live].sum(axis=0)
                   + (nv + 2) * U * np.abs(g * lines).sum(axis=0))
            fading = (np.abs(g) * np.abs(lines))[~live].sum(axis=0)
            err = np.abs(rows[e].astype(np.float64) - want)
            if (err > tol + fading).any():
                i = int(np.argmax(err - tol - fading))
                bad.append(f"scale update {u} ear {e}: {int((err > tol + fading).sum())} samples outside, "
                           f"at {i}: err {err[i]:.3e} bound {tol[i] + fading[i]:.3e}")
    _assert_ok(bad)
