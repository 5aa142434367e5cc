"""The convolution effect slot in isolation, against a float64 model.

A slot's output is linear in its input, so the exact answer is cheap: every line is the float64
convolution of the float32 input (its whole history since the slot was installed) with the
float32 IR, mixed into Dry with the output gains restated in float64.  The harness feeds each
convolution slot an exact input and reads back only the slot's output:

  - the device has no voices and no post-process (POST_NONE: RealOut is the Dry mix);
  - between render_begin and render_end the test writes the slot's input into wet channel 0
    and loud noise into wet channels 1..cw-1, which a convolution slot must ignore
    (ConvolutionState::process reads channel 0 only, alc/effects/convolution.cpp:636).

The same script drives the CUDA library, the CPU oracle, and the model (with or without a
deliberate defect, to show the bound would catch it).

Bound.  Per output sample, |kernel - model| <= C_BOUND * 2^-24 * B[n], with B the sum over the
lines mixed into that output of |gain| * S[n] and

    S[n] = sum_{k<128} |h_k| |x_{n-k}|  +  sum_s ||h_s||_2 (||x_{j-1-s}||_2 + ||x_{j-2-s}||_2)

h_s is segment s of the IR (taps [128(s+1), 128(s+2))), x_b input block b on the slot's 128-sample
grid, j the block holding n.  The segments' share is block-wide because FFT rounding spreads over
a whole block; by Cauchy-Schwarz S[n] >= |y[n]|, so S also bounds the rounding of the gain and of
the Dry sum.  A slot that targets another convolution slot hands its error envelope on as part of
the target's input.
"""
import ctypes as C

import numpy as np
from scipy.signal import fftconvolve

from helpers.mixlib import MixDevice
from pyb200mix import abi

U = 2.0 ** -24
# One constant for every case.  Worst err / (2^-24 S) seen on an H100 80GB HBM3 (132 SMs, 700 W
# power limit): 3.86 (every IR length to 20 000 taps), 2.26 (conv -> conv), 1.47 (480 000 taps),
# 0.08 (32 x 96 000 taps); the CPU oracle stays under 2.  The defects the CPU file applies to
# the model land at 587x C or more.
C_BOUND = 16.0
BLOCK = 128                     # kConvBlock        (csrc/effect_kernels.cuh:25)
WINDOW = 9                      # kConvMaxBlocks    (csrc/effect_kernels.cuh:27), the MAC's s mod 9 window
MAX_CHUNKS = 48                 # kConvMaxChunks    (csrc/effect_kernels.cuh:28)
STAGES = 3                      # kConvStages       (csrc/effect_kernels.cuh:585)
K_EPS = np.float32(1.1920929e-07)   # kEps          (csrc/mixer_kernels.cuh:39)
K_SILENCE = np.float32(0.00001)     # kSilence      (csrc/mixer_kernels.cuh:38)
NOISE = 64.0                    # amplitude of what goes into the wet channels a slot must ignore
F32 = np.float32


def nseg(taps):
    """mNumConvolveSegs (b200mix_slot_convolution; convolution.cpp:375-376)."""
    return max(-(-taps // BLOCK), 2) - 1


# ---- the host's chunk plan ---------------------------------------------------------------

def conv_chunks(slots, sms):
    """SlotTable::refresh (csrc/slot_table.hpp:445-450): slots = [(segs, channels)] of the
    installed convolution slots."""
    work = sum(ch for _, ch in slots)
    segs = max(s for s, _ in slots)
    return max(1, min(MAX_CHUNKS, (segs + 17) // 18, (4 * sms + work - 1) // work))


def chunk_plan(segs, chunks):
    """k_conv_mac's segment ranges for one slot (conv_chunk_len, effect_kernels.cuh:501;
    zcnt as in k_conv_ifft; rounds of 9 aligned segments as in k_conv_mac)."""
    clen = -(-segs // chunks)
    zcnt = -(-segs // clen)
    starts = [z * clen for z in range(zcnt)]
    rounds = max(-(-(min(s0 + clen, segs) - (s0 - s0 % WINDOW)) // WINDOW) for s0 in starts)
    return {"segs": segs, "clen": clen, "zcnt": zcnt, "starts": starts, "rounds": rounds}


CATEGORIES = ("chunks==1", "chunks==48", "clen%9==0", "clen%9!=0", "clen<9 start%9!=0", "clen==1",
              "empty chunks beside a long slot", "zcnt<chunks", "rounds>stages")


def categories(slots, sms):
    """The chunk-plan categories one set of installed slots reaches on `sms` SMs."""
    chunks = conv_chunks(slots, sms)
    plans = [chunk_plan(s, chunks) for s, _ in slots]
    got = set()
    if chunks == 1:
        got.add("chunks==1")
    if chunks == MAX_CHUNKS:
        got.add("chunks==48")
    for p in plans:
        got.add("clen%9==0" if p["clen"] % WINDOW == 0 else "clen%9!=0")
        if p["clen"] < WINDOW and any(s0 % WINDOW for s0 in p["starts"]):
            got.add("clen<9 start%9!=0")
        if p["clen"] == 1:
            got.add("clen==1")
        if p["zcnt"] < chunks:
            got.add("zcnt<chunks")
            if any(q["zcnt"] == chunks for q in plans):
                got.add("empty chunks beside a long slot")
        if p["rounds"] > STAGES:
            got.add("rounds>stages")
    return chunks, plans, got


# ---- scripts -----------------------------------------------------------------------------

class Script:
    """A device's life: installs, targets, gains, disables and updates with their wet input."""

    def __init__(self, name, dry, cw, slots, seed):
        self.name, self.dry, self.cw, self.slots = name, dry, cw, slots
        self.rng = np.random.default_rng(seed)
        self.ops = []
        self.frames = 0

    def install(self, sl, ir, gains):
        ir = np.ascontiguousarray(np.atleast_2d(ir), dtype=F32)
        self.ops.append(("install", sl, ir, np.atleast_2d(gains).astype(F32)))

    def target(self, sl, tgt):
        self.ops.append(("target", sl, tgt))

    def gains(self, sl, g):
        self.ops.append(("gains", sl, np.atleast_2d(g).astype(F32)))

    def disable(self, sl):
        self.ops.append(("disable", sl))

    def update(self, n, inputs):
        """inputs: {slot: float32[n]} for wet channel 0; the other wet channels get noise."""
        wet = np.zeros((self.slots, self.cw, n), dtype=F32)
        if self.cw > 1:
            wet[:, 1:] = (self.rng.uniform(-NOISE, NOISE, (self.slots, self.cw - 1, n))).astype(F32)
        for sl, x in inputs.items():
            wet[sl, 0] = x
        self.ops.append(("update", n, wet))
        self.frames += n

    def slot_sets(self):
        """Every distinct set of installed slots an update of this script ran with."""
        inst, sets = {}, []
        for op in self.ops:
            if op[0] == "install":
                inst[op[1]] = (nseg(op[2].shape[1]), op[2].shape[0])
            elif op[0] == "disable":
                inst.pop(op[1], None)
            elif op[0] == "update":
                s = tuple(v for _, v in sorted(inst.items()))
                if s and s not in sets:
                    sets.append(s)
        return sets


# ---- the harness ---------------------------------------------------------------------------

def device_desc(dry, cw, slots):
    d = abi.DeviceDesc()
    d.struct_size = C.sizeof(abi.DeviceDesc)
    d.cuda_device = -1
    d.sample_rate = 48000
    d.dry_channels = dry
    d.real_channels = dry                   # POST_NONE: RealOut is the Dry mix
    d.wet_channels = cw
    d.num_sends = 1
    d.ir_size = 0
    d.post_process = abi.POST_NONE
    d.max_voices = 1
    d.max_buffers = 1
    d.max_slots = slots
    return d


def _cuda_view(ptr, count):
    import torch

    class _W:
        pass
    w = _W()
    w.__cuda_array_interface__ = {"shape": (count,), "typestr": "<f4", "data": (ptr, False), "version": 2}
    return torch.as_tensor(w, device=torch.device("cuda", 0))


def run(script, lib):
    """Runs the script on one implementation; returns RealOut [dry][frames] (float32)."""
    gpu = lib.prefix == "b200mix_"
    if gpu:
        import torch
    dev = MixDevice(lib, device_desc(script.dry, script.cw, script.slots))
    outs = []
    try:
        for op in script.ops:
            kind = op[0]
            if kind == "install":
                dev.slot_convolution(op[1], op[2], op[3])
            elif kind == "target":
                dev.slot_target(op[1], op[2])
            elif kind == "gains":
                rc = lib.slot_output_gains(dev.h, op[1], op[2].shape[0], np.ascontiguousarray(op[2]).ctypes.data)
                assert rc == 0, rc
            elif kind == "disable":
                assert lib.slot_disable(dev.h, op[1]) == 0
            else:
                n, wet = op[1], op[2]
                ptr, cnt = dev.render_begin(n)
                assert cnt == script.slots * script.cw * abi.LINE
                host = np.zeros((script.slots, script.cw, abi.LINE), dtype=F32)
                host[:, :, :n] = wet
                if gpu:
                    torch.cuda.synchronize()         # the library's stream has cleared the wet buffers
                    _cuda_view(ptr, cnt).copy_(torch.from_numpy(host.reshape(-1)))
                    torch.cuda.synchronize()
                else:
                    np.ctypeslib.as_array((C.c_float * cnt).from_address(ptr))[:] = host.reshape(-1)
                outs.append(dev.render_end())
    finally:
        dev.close()
    return np.concatenate(outs, axis=1)


# ---- the float64 model ---------------------------------------------------------------------

DEFECTS = ("drop last segment", "drop one chunk", "head one tap late", "one segment one block late",
           "spectrum ring one slot off", "fifo phase off by one", "gain ramp indexed i+1",
           "wet channel 1 leaks in at 1e-3")


def _shift(y, d):
    out = np.zeros_like(y)
    if d < len(y):
        out[d:] = y[:len(y) - d]
    return out


def line(h, x, defect=None, chunk=None):
    """float64 h * x over the instance's history (head by direct sum, the rest by FFT)."""
    T = len(x)
    h = h.astype(np.float64)
    ns = nseg(len(h))
    tail = np.zeros(BLOCK * (ns + 2))
    tail[BLOCK:len(h)] = h[BLOCK:]
    if defect == "drop last segment":
        tail[BLOCK * ns:BLOCK * (ns + 1)] = 0.0
    elif defect == "drop one chunk" and chunk is not None:
        s0, s1 = chunk
        tail[BLOCK * (s0 + 1):BLOCK * (s1 + 1)] = 0.0
    elif defect == "one segment one block late":
        s = ns // 2
        seg = tail[BLOCK * (s + 1):BLOCK * (s + 2)].copy()
        tail[BLOCK * (s + 1):BLOCK * (s + 2)] = 0.0
        tail[BLOCK * (s + 2):BLOCK * (s + 3)] += seg
    yh = np.convolve(x, h[:BLOCK])[:T]
    yt = fftconvolve(x, tail)[:T] if tail.any() else np.zeros(T)
    if defect == "head one tap late":
        yh = _shift(yh, 1)
    elif defect == "spectrum ring one slot off":
        yt = _shift(yt, BLOCK)
    elif defect == "fifo phase off by one":
        yt = _shift(yt, 1)
    return yh + yt


def envelope(h, a):
    """S[n] for IR h and a non-negative input envelope a, on a's own 128-sample grid."""
    T = len(a)
    h = h.astype(np.float64)
    ns = nseg(len(h))
    hp = np.zeros(BLOCK * (ns + 1))
    hp[:len(h)] = h
    sh = np.convolve(a, np.abs(hp[:BLOCK]))[:T]
    hs = np.sqrt((hp[BLOCK:].reshape(ns, BLOCK) ** 2).sum(axis=1))
    nb = -(-T // BLOCK)
    ap = np.zeros(nb * BLOCK)
    ap[:T] = a
    e = np.sqrt((ap.reshape(nb, BLOCK) ** 2).sum(axis=1))
    ae = np.convolve(hs, e)[:nb]                        # ae[m] = sum_s ||h_s|| ||x_{m-s}||
    tj = np.zeros(nb)
    tj[1:] += ae[:nb - 1]
    tj[2:] += ae[:nb - 2]
    return sh + np.repeat(tj, BLOCK)[:T]


def gain_rows(cur, tgt, n, defect=None):
    """MixSamples with Counter = samplesToDo as k_slot_output_mix / k_slot_target_mix run it
    (effect_kernels.cuh:862-873, 897-910): step = (target - current) * (1/n) in float32; the
    ramp current + step*i for i < n when |step| > kEps, else the target when |target| > kSilence,
    else nothing.  Returns (gain [lines][width][n] float64, |gain| scale for the bound)."""
    delta = F32(1.0) / F32(n)
    step = ((tgt - cur).astype(F32) * delta).astype(F32)
    ramp = np.abs(step) > K_EPS
    flat = np.where(np.abs(tgt) > K_SILENCE, tgt, F32(0)).astype(np.float64)
    i = np.arange(n, dtype=np.float64) + (1.0 if defect == "gain ramp indexed i+1" else 0.0)
    g = np.where(ramp[..., None], cur.astype(np.float64)[..., None] + step.astype(np.float64)[..., None] * i,
                 flat[..., None])
    # the float32 ramp rounds relative to its end points, not to the gain at sample i
    scale = np.where(ramp, np.maximum(np.abs(cur), np.abs(tgt)), np.abs(flat)).astype(np.float64)
    return g, scale


class _Instance:
    def __init__(self, sl, ir, t0, target):
        self.sl, self.ir, self.t0, self.t1, self.target = sl, ir, t0, None, target
        self.updates = []                 # (t, n, cur, tgt)
        self.cur = np.zeros((ir.shape[0], 0), dtype=F32)
        self.tgt = None


def model(script, defect=None, chunk=None, spot_check=True):
    """(Dry [dry][frames] float64, bound B [dry][frames]): the exact mix and the sum of
    |gain| * S over the lines mixed into each output sample."""
    T = script.frames
    inj = np.zeros((script.slots, T))
    leak = np.zeros((script.slots, T))
    targets = [abi.NO_SLOT] * script.slots
    live, done = {}, []
    t = 0
    for op in script.ops:
        kind = op[0]
        if kind == "install":
            if op[1] in live:
                live[op[1]].t1 = t
                done.append(live[op[1]])
            inst = _Instance(op[1], op[2], t, targets[op[1]])
            inst.tgt = op[3]
            inst.cur = np.zeros_like(op[3])
            live[op[1]] = inst
        elif kind == "target":
            targets[op[1]] = op[2]
            if op[1] in live:
                live[op[1]].target = op[2]
        elif kind == "gains":
            live[op[1]].tgt = op[2]
            if live[op[1]].cur.shape != op[2].shape:
                live[op[1]].cur = np.zeros_like(op[2])
        elif kind == "disable":
            live[op[1]].t1 = t
            done.append(live.pop(op[1]))
        else:
            n, wet = op[1], op[2]
            inj[:, t:t + n] = wet[:, 0]
            if script.cw > 1:
                leak[:, t:t + n] = wet[:, 1]
            for inst in live.values():
                inst.updates.append((t, n, inst.cur.copy(), inst.tgt.copy()))
                inst.cur = inst.tgt.copy()            # k_slot_gains_commit: Current <- Target
            t += n
    for inst in live.values():
        inst.t1 = T
        done.append(inst)

    def depth(inst):
        d, s = 0, inst.target
        while s != abi.NO_SLOT and d <= script.slots:
            d, s = d + 1, targets[s]
        return d
    # every slot before its target (alc/alu.cpp:2211-2251)
    done.sort(key=lambda i: -depth(i))
    dry = np.zeros((script.dry, T))
    bound = np.zeros((script.dry, T))
    x_in = inj.copy()
    if defect == "wet channel 1 leaks in at 1e-3":
        x_in += 1e-3 * leak
    env_in = np.zeros((script.slots, T))
    for inst in done:
        t0, t1 = inst.t0, inst.t1
        if t1 <= t0:
            continue
        x = x_in[inst.sl, t0:t1]
        a = np.abs(x)
        e_in = env_in[inst.sl, t0:t1]
        ys, ss = [], []
        for c in range(inst.ir.shape[0]):
            h = inst.ir[c]
            y = line(h, x, defect, chunk)
            if spot_check and defect is None:
                _spot_check(h, x, y)
            s = envelope(h, a)
            if e_in.any():
                s = s + envelope(h, e_in)
            ys.append(y)
            ss.append(s)
        to_dry = inst.target == abi.NO_SLOT
        for (tu, n, cur, tgt) in inst.updates:
            g, sc = gain_rows(cur, tgt, n, defect)
            lo, hi = tu - t0, tu - t0 + n
            for c in range(len(ys)):
                contrib = g[c] * ys[c][lo:hi]
                env = sc[c][:, None] * ss[c][lo:hi]
                if to_dry:
                    dry[:, tu:tu + n] += contrib[:script.dry]
                    bound[:, tu:tu + n] += env[:script.dry]
                else:
                    # the target reads its wet channel 0 only
                    x_in[inst.target, tu:tu + n] += contrib[0]
                    env_in[inst.target, tu:tu + n] += env[0]
    return dry, bound


def _spot_check(h, x, y, count=48):
    """The FFT convolution against a direct float64 sum on a subsample of outputs."""
    T = len(x)
    if T == 0:
        return
    rng = np.random.default_rng(T + len(h))
    idx = np.unique(np.concatenate([rng.integers(0, T, count), [T - 1]]))
    hr = h.astype(np.float64)[::-1].copy()            # hr[L-1-k] = h[k]
    floor = 1e-13 * float(np.abs(y).max())
    for n in idx:
        m = min(len(hr), n + 1)
        seg = x[n - m + 1:n + 1]
        prod = hr[len(hr) - m:] * seg
        ref, mag = float(prod.sum()), float(np.abs(prod).sum())
        assert abs(ref - y[n]) <= 1e-12 * mag + floor, (n, ref, y[n])


def ratio(out, ref, bound):
    """Worst |out - ref| / (2^-24 * B), after the float64 model's own error (1e-13 of the case's
    peak: FFT noise where the exact answer is zero)."""
    floor = 1e-13 * float(np.abs(ref).max())
    err = np.maximum(np.abs(out.astype(np.float64) - ref) - floor, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err > 0, err / (U * bound), 0.0)
    return float(r.max())


def check(script, out, what=""):
    """Holds a run's RealOut to the model; returns the worst ratio."""
    ref, bound = model(script)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    assert np.abs(ref).max() > 1e-3, f"{script.name}: the slots' output is silent"
    r = ratio(out, ref, bound)
    assert r <= C_BOUND, f"{script.name}{what}: err/(2^-24 S) = {r:.3g} > {C_BOUND}"
    return r


# ---- inputs --------------------------------------------------------------------------------

def flat_ir(rng, channels, taps, rising=False):
    """Every segment carries comparable energy (rising: the last segment dominates)."""
    env = np.ones(taps) if not rising else np.exp(3.0 * np.arange(taps) / max(taps - 1, 1))
    h = rng.standard_normal((channels, taps)) * env
    return (h / np.sqrt((h ** 2).sum(axis=1, keepdims=True))).astype(F32)


def tagged_ir(rng, channels, taps):
    """One non-zero tap per segment (and one in the head), at a position that moves with the
    segment and the channel: a misplaced segment or block shows up where it lands."""
    h = np.zeros((channels, taps), dtype=F32)
    for c in range(channels):
        h[c, (7 * c + 3) % min(BLOCK, taps)] = F32(0.5 + 0.5 * rng.random())
        for s in range(nseg(taps)):
            k = BLOCK * (s + 1) + (37 * s + 11 * c + 5) % BLOCK
            if k < taps:
                h[c, k] = F32((0.3 + 0.7 * rng.random()) * (-1) ** (s + c))
    return h


def white(rng, n, amp=1.0):
    return rng.uniform(-amp, amp, n).astype(F32)


def static_gains(rng, channels, width):
    return (rng.uniform(-1.0, 1.0, (channels, width))).astype(F32)


def next_gains(rng, prev, k, n):
    """The output gains of update k (of n frames) in a schedule that changes them every
    update, given the previous targets: to 0 and from 0, sign flips, targets 2 % above and
    below kSilence, and float32 steps 3 % above and below kEps (from small gains, where the
    float32 grid is fine enough to place them)."""
    kind = k % 9
    g = rng.uniform(-1.0, 1.0, prev.shape).astype(F32)
    if kind == 1:
        g[:, ::2] = 0.0                                  # to 0 (kind 2: from 0)
    elif kind == 3:
        g = -prev                                        # sign flip
    elif kind in (4, 5):
        g[:, ::2] = F32(K_SILENCE * (1.02 if kind == 4 else 0.98)) * np.where(prev[:, ::2] < 0, -1, 1)
    elif kind == 6:
        g = (g * F32(1e-3)).astype(F32)
    elif kind in (7, 8):
        step = (1.03 if kind == 7 else 0.97) * float(K_EPS)
        g = (prev + F32(step * n) * np.where(rng.random(prev.shape) < 0.5, -1, 1)).astype(F32)
    return g.astype(F32)


# ---- the cases -----------------------------------------------------------------------------

UPDATE_SIZES = (1, 2, 127, 128, 129, 255, 256, 1023, 1024)
IR_LENGTHS = (1, 2, 127, 128, 129, 255, 256, 257, 384, 385, 1152, 1153, 1281, 2305, 2433, 12801, 20000)


def wrap_frames(taps, times):
    """Samples for the input-spectrum ring (segs + 9 blocks) to go round `times` times."""
    return times * (nseg(taps) + WINDOW) * BLOCK


def _ragged(script, frames, inputs_fn, sizes=UPDATE_SIZES, k0=0):
    k = k0
    while frames > 0:
        n = sizes[k % len(sizes)]
        script.update(n, inputs_fn(n))
        frames -= n
        k += 1
    return k


def case_lengths(max_taps=20000, dry=16, seed=1):
    """Every IR length up to max_taps on one device, IR channels cycling 1/2/4/8/16, flat
    envelopes (one rising), ragged update sizes, twice round the longest slot's ring."""
    lengths = [t for t in IR_LENGTHS if t <= max_taps]
    s = Script(f"lengths<={max_taps}", dry=dry, cw=2, slots=len(lengths), seed=seed)
    rng = s.rng
    for sl, taps in enumerate(lengths):
        ch = (1, 2, 4, 8, 16)[sl % 5]
        s.install(sl, flat_ir(rng, ch, taps, rising=(taps == 1281)), static_gains(rng, ch, dry))
    _ragged(s, wrap_frames(max(lengths), 2),
            lambda n: {sl: white(rng, n) for sl in range(len(lengths))})
    return s


def case_long(seed=2):
    """480 000 taps (3749 segments: the 48-chunk cap, chunks of 79 off the 9-grid, rounds > 3)
    with a 432-segment slot (clen 9), a 100-segment slot (clen 3) and a 9-segment slot (clen 1,
    empty chunks) beside it; once round the long ring, 128 consecutive 1023-frame updates."""
    s = Script("long 480000 taps", dry=4, cw=2, slots=4, seed=seed)
    rng = s.rng
    spec = [(480000, 2, False), (BLOCK * 433, 1, True), (12801, 1, False), (1153, 1, False)]
    for sl, (taps, ch, rising) in enumerate(spec):
        s.install(sl, flat_ir(rng, ch, taps, rising), static_gains(rng, ch, s.dry))
    frames = wrap_frames(480000, 1)
    k = _ragged(s, 520, lambda n: {sl: white(rng, n) for sl in range(4)}, sizes=(1, 2, 127, 129, 255, 6))
    frames -= 520
    _ragged(s, 128 * 1023, lambda n: {sl: white(rng, n) for sl in range(4)}, sizes=(1023,), k0=k)
    frames -= 128 * 1023
    _ragged(s, frames, lambda n: {sl: white(rng, n) for sl in range(4)}, sizes=(1024,))
    return s


def case_bench(seed=3):
    """tools/bench_effects.py --effect conv's shape: 32 mono slots of 96 000 taps (749
    segments), the widest Dry mix (32 channels), half the slots at about 1e3 amplitude; once
    round the ring."""
    s = Script("32 x 96000 taps mono", dry=32, cw=2, slots=32, seed=seed)
    rng = s.rng
    for sl in range(32):
        s.install(sl, flat_ir(rng, 1, 96000, rising=(sl == 5)), static_gains(rng, 1, 32))
    amp = [1.0 if sl % 2 else 1e3 for sl in range(32)]
    _ragged(s, wrap_frames(96000, 1), lambda n: {sl: white(rng, n, amp[sl]) for sl in range(32)},
            sizes=(1024,))
    return s


def _impulses(n, t):
    """Unit impulses at block offsets 0, 1, 127 and 128 of every other 3-block group on the
    slot's grid (t = the update's first sample on that grid), and at the last sample of the
    update (of every 7th, for 1-frame updates)."""
    p = t + np.arange(n)
    x = ((p // (3 * BLOCK)) % 2 == 0) & np.isin(p % (3 * BLOCK), (0, 1, 127, 128))
    x = x.astype(F32)
    if n > 1 or t % 7 == 0:
        x[n - 1] = 1.0
    return x


def case_tagged(seed=4, one_frame_updates=300):
    """Segment-tagged IRs driven by unit impulses: a 16-channel slot beside a 1-channel one
    (k_conv_mac's blockIdx.y >= channels early return), runs of 1-frame updates (no block
    completes: only the head and the FIFO carry work), then ragged updates, twice round."""
    s = Script("segment-tagged", dry=4, cw=4, slots=2, seed=seed)
    rng = s.rng
    spec = [(2433, 16), (1153, 1)]
    for sl, (taps, ch) in enumerate(spec):
        s.install(sl, tagged_ir(rng, ch, taps), static_gains(rng, ch, s.dry))
    t = [0]

    def inputs(n):
        x = _impulses(n, t[0])
        t[0] += n
        return {0: x, 1: x}
    _ragged(s, one_frame_updates, inputs, sizes=(1,))
    _ragged(s, wrap_frames(2433, 2), inputs)
    _ragged(s, 200, inputs, sizes=(1,))
    _ragged(s, 3 * 1024, inputs)
    return s


def case_gains(seed=5):
    """Three slots of different lengths, output gains changed every update: from and to 0,
    sign flips, float32 steps 3 % above and below kEps, targets 2 % above and below kSilence."""
    s = Script("gains every update", dry=4, cw=2, slots=3, seed=seed)
    rng = s.rng
    spec = [(385, 2), (1281, 1), (2305, 4)]
    tg = {}
    for sl, (taps, ch) in enumerate(spec):
        tg[sl] = static_gains(rng, ch, s.dry)
        s.install(sl, flat_ir(rng, ch, taps), tg[sl])
    k = 0
    frames = wrap_frames(2305, 2)
    while frames > 0:
        n = UPDATE_SIZES[(k * 5) % len(UPDATE_SIZES)]
        for sl in range(3):
            tg[sl] = next_gains(rng, tg[sl], k, n)
            s.gains(sl, tg[sl])
        s.update(n, {sl: white(rng, n) for sl in range(3)})
        frames -= n
        k += 1
    return s


def case_lifecycle(seed=6):
    """A running slot re-installed with another IR length (the model restarts from zero
    history), a slot disabled and installed again; twice round each ring every time."""
    s = Script("re-install / disable", dry=4, cw=2, slots=3, seed=seed)
    rng = s.rng
    s.install(0, flat_ir(rng, 2, 1153), static_gains(rng, 2, 4))
    s.install(1, flat_ir(rng, 1, 2305), static_gains(rng, 1, 4))
    feed = lambda n: {0: white(rng, n), 1: white(rng, n), 2: white(rng, n)}  # noqa: E731
    _ragged(s, wrap_frames(2305, 2) + 77, feed)
    s.install(0, flat_ir(rng, 1, 257, rising=True), static_gains(rng, 1, 4))
    _ragged(s, wrap_frames(2305, 2), feed, sizes=(129, 1023, 1, 255))
    s.disable(1)
    _ragged(s, 3000, feed)
    s.install(1, flat_ir(rng, 4, 1281), static_gains(rng, 4, 4))
    s.install(2, flat_ir(rng, 1, 385), static_gains(rng, 1, 4))
    _ragged(s, wrap_frames(1281, 2) + 500, feed)
    return s


def case_chain(seed=7):
    """A convolution slot whose output goes to another convolution slot's Wet input
    (two stages, k_slot_target_mix), with a third slot straight to Dry; gains change every
    update on the first hop."""
    s = Script("conv -> conv", dry=4, cw=4, slots=3, seed=seed)
    rng = s.rng
    s.install(0, flat_ir(rng, 2, 1281), static_gains(rng, 2, 4))
    s.target(0, 1)
    tg = static_gains(rng, 2, s.cw)
    s.gains(0, tg)
    s.install(1, flat_ir(rng, 1, 2305), static_gains(rng, 1, 4))
    s.install(2, flat_ir(rng, 1, 129), static_gains(rng, 1, 4))
    k, frames = 0, wrap_frames(2305, 2)
    while frames > 0:
        n = UPDATE_SIZES[(k * 4) % len(UPDATE_SIZES)]
        if k:
            tg = next_gains(rng, tg, k, n)
            s.gains(0, tg)
        s.update(n, {0: white(rng, n), 1: white(rng, n, 0.25), 2: white(rng, n)})
        frames -= n
        k += 1
    return s


GPU_CASES = (case_lengths, case_long, case_bench, case_tagged, case_gains, case_lifecycle, case_chain)
ORACLE_CASES = (lambda: case_lengths(max_taps=2433, dry=4), case_tagged, case_gains, case_lifecycle, case_chain)
