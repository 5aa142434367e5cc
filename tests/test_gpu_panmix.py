"""The tensor-core pan-mix (k_panmix_tc, openal-soft_b200/csrc/panmix_tc.cuh), which sums the dry
bus of every parked (non-HRTF) voice past the gain fades on devices with 5..16 dry channels.

(1) Kernel level: the kernel alone (openal-soft_b200/libpanmix_probe.so, built from
    tests/native/panmix_probe.cu with the library's flags) against a float64 sum of the same
    products, at every bus width the mixer uses, at entry counts that leave 0..7 entries in the
    last K block and empty trailing chunks, with gathered and deferred lines and inputs chosen to
    stress the 3xTF32 split; plus the exact footprint of its writes.
(2) Library level: seeded scenes through the C ABI against the CPU oracle, each run twice on the
    product — on the tensor cores and with B200MIX_PANMIX_SIMT=1 — where the difference in launch
    counts proves the kernel ran on every full update and on no ragged one."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

PROBE_SO = os.path.join(mixlib.ROOT, "openal-soft_b200", "libpanmix_probe.so")
LINE, FADE = abi.LINE, 128               # samples 0..127 belong to k_send_mix's first (fade) tile
K = 8                                    # voices per MMA (kPmK)
CHUNKS_MAX = 128                         # kDryChunksMax
SI_DEFERRED = 4                          # kSiDeferred
SENTINEL = np.int32(0x7FBADBAD)          # a NaN: any sum that reads it, or a write over it, shows
GUARD = 4096                             # floats after the partial rows that nothing may touch

_probe = None


def probe():
    global _probe
    if _probe is None:
        lib = C.CDLL(PROBE_SO)
        lib.panmix_probe_run.restype = C.c_int
        lib.panmix_probe_run.argtypes = [C.c_void_p] * 6 + [C.c_uint32, C.c_uint32, C.c_void_p]
        _probe = lib
    return _probe


def chunking(n):
    """The entry ranges of the dry-bus launch (b200mix.cu: chunks of 64 entries, at most 128
    CTAs; k_panmix_tc splits [0, n) into `chunks` ranges of ceil(n / chunks))."""
    chunks = max(1, min(CHUNKS_MAX, (n + 63) // 64))
    per = -(-n // chunks)
    return chunks, [(min(z * per, n), min(min(z * per, n) + per, n)) for z in range(chunks)]


# ---------------------------------------------------------------------------------------------
# (1) kernel level
#
# Tolerance.  Each product x*g goes through the tensor cores as  xh*gh + xl*gh + xh*gl  where
# xh = x rounded to tf32 (|x - xh| <= 2^-11 |x|) and xl = (x - xh) truncated to tf32
# (|x - xh - xl| < 2^-10 |x - xh| <= 2^-21 |x|), the same for g.  The products of tf32 operands
# are exact in fp32, so what is lost per product is the dropped xl*gl (<= 2^-22 |xg|) and the two
# truncated tails (<= 2^-21 |xg| each): at most 5 * 2^-22 |xg|.  On top of that the fp32
# accumulators take three MMAs per K block of 8 entries, each rounding (or truncating) once
# against a running sum no larger than the chunk's sum of |products|: 3 * nkb * 2^-23 of it, with
# nkb = ceil(entries of the chunk / 8).  So, per chunk, channel and sample,
#       |got - ref| <= (5 * 2^-22 + 3 * nkb * 2^-23) * sum_e |g_e x_e|.
# Normalising by sum |g x| rather than by the peak keeps cancelling sums judged.  A 1xTF32 kernel
# (or one without either lo term) is off by ~2^-12 per product, several times this bound even at
# the largest chunk, and far outside it at small ones.
def _tolerance(nkb):
    return 5.0 * 2.0 ** -22 + 3.0 * nkb * 2.0 ** -23


def _inputs(kind, cw, n, seed):
    """(entry voices [n], sendinfo [nvoices], xscratch, dline or None, geff [n][cw]) as numpy."""
    rng = np.random.default_rng(seed)
    nvoices = n + 17                     # a few voices no entry refers to
    if kind == "cancelling":
        # pairs of entries on the same line with opposite gains: the exact sum is 0 (plus the
        # unpaired last entry of an odd count)
        vids = rng.permutation(nvoices)[:(n + 1) // 2]
        voices = np.repeat(vids, 2)[:n]
    else:
        voices = rng.permutation(nvoices)[:n]            # a gather, not a stream
    deferred = rng.random(nvoices) < 0.35
    # the kernel may look at nothing but the deferred bit of sendinfo
    info = (rng.integers(0, 1 << 16, nvoices).astype(np.uint32) & ~np.uint32(SI_DEFERRED)) \
        | np.where(deferred, SI_DEFERRED, 0).astype(np.uint32)

    def values(shape):
        u = rng.uniform(-1.0, 1.0, shape).astype(np.float32)
        if kind == "mantissa":
            # low 13 bits all set: the tf32 hi part rounds up, the lo part is negative
            b = u.view(np.uint32) | np.uint32(0x1FFF)
            u = b.view(np.float32)
        elif kind == "tf32_exact":
            u = (u.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
        return u

    x = values((nvoices, LINE))
    d = values((nvoices, LINE))
    if kind == "magnitudes":
        x *= (10.0 ** rng.uniform(-5.0, 0.0, (nvoices, 1))).astype(np.float32)
        d *= (10.0 ** rng.uniform(-5.0, 0.0, (nvoices, 1))).astype(np.float32)
    g = values((n, cw)) * np.float32(0.5)
    if kind == "cancelling":
        g[1::2] = -g[0::2][:n // 2]
    use_dline = kind != "no_dline"
    # what the kernel must not read is NaN: the fade tile of every line, the deferred voices'
    # xscratch rows and the other voices' dline rows (with no dline, xscratch serves everyone)
    x[:, :FADE] = np.nan
    d[:, :FADE] = np.nan
    if use_dline:
        x[deferred, FADE:] = np.nan
        d[~deferred, FADE:] = np.nan
    lines = np.where(deferred[:, None], d, x) if use_dline else x
    return voices, info, x, (d if use_dline else None), g, lines


KINDS = ("uniform", "no_dline", "mantissa", "tf32_exact", "magnitudes", "cancelling")
WORST = {}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [65, 100, 130, 1000, 4096, 8193, 9000])
@pytest.mark.parametrize("cw", [5, 7, 9, 12, 16])
def test_panmix_kernel_vs_float64(cw, n, kind):
    import torch
    voices, info, x, d, g, lines = _inputs(kind, cw, n, seed=cw * 100003 + n * 7 + KINDS.index(kind))
    chunks, ranges = chunking(n)
    dev = torch.device("cuda", 0)
    t_ss = torch.tensor([0, n], dtype=torch.int32, device=dev)
    ent = np.zeros((n, 2), dtype=np.uint32)
    ent[:, 0] = voices
    t_ent = torch.from_numpy(ent.view(np.int32)).to(dev)
    t_info = torch.from_numpy(info.view(np.int32)).to(dev)
    t_x = torch.from_numpy(x).to(dev)
    t_d = torch.from_numpy(d).to(dev) if d is not None else None
    t_g = torch.from_numpy(g).to(dev)
    rows = chunks * cw * LINE
    t_part = torch.full((rows + GUARD,), int(SENTINEL), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    rc = probe().panmix_probe_run(t_ss.data_ptr(), t_ent.data_ptr(), t_info.data_ptr(), t_x.data_ptr(),
                                  t_d.data_ptr() if t_d is not None else None, t_g.data_ptr(),
                                  cw, chunks, t_part.data_ptr())
    assert rc == 0, f"panmix_probe_run -> cudaError {rc}"
    raw = t_part.cpu().numpy()

    # write footprint: the fade tile of every row and everything past the rows stay untouched
    assert (raw[rows:] == SENTINEL).all(), "k_panmix_tc wrote past its partial rows"
    part_i = raw[:rows].reshape(chunks, cw, LINE)
    assert (part_i[:, :, :FADE] == SENTINEL).all(), "k_panmix_tc wrote into samples 0..127"
    assert not (part_i[:, :, FADE:] == SENTINEL).any(), "k_panmix_tc left samples 128..1023 unwritten"
    part = part_i[:, :, FADE:].view(np.float32).astype(np.float64)

    X = lines[voices, FADE:].astype(np.float64)           # [n][896]
    G = g.astype(np.float64)                              # [n][cw]
    worst = 0.0
    empty = 0
    for z, (e0, e1) in enumerate(ranges):
        if e0 == e1:
            # an empty chunk (nkb == 0) still owns its rows: zeros, so the reduction can sum them
            assert (part_i[z, :, FADE:] == 0).all(), f"empty chunk {z} did not write zeros"
            empty += 1
            continue
        ref = G[e0:e1].T @ X[e0:e1]
        mag = np.abs(G[e0:e1]).T @ np.abs(X[e0:e1])
        err = np.abs(part[z] - ref) / mag
        tol = _tolerance(-(-(e1 - e0) // K))
        bad = ~(err <= tol)
        if bad.any():
            c, i = np.argwhere(bad)[0]
            pytest.fail(f"cw {cw} n {n} {kind}: chunk {z} [{e0}, {e1}) channel {c} sample {FADE + i}: "
                        f"got {part[z, c, i]:.9g} ref {ref[c, i]:.9g} |err|/sum|gx| {err[c, i]:.3e} > {tol:.3e}")
        worst = max(worst, float(err.max()))
    # the chunking really has the shape this entry count was picked for
    assert empty == sum(e0 == e1 for e0, e1 in ranges)
    if n in (8193, 9000):
        assert empty >= 1
    WORST[cw] = max(WORST.get(cw, 0.0), worst)
    print(f"panmix cw={cw} n={n} {kind}: worst |err|/sum|gx| = {worst:.3e} (running worst for cw {cw}: "
          f"{WORST[cw]:.3e})")


# ---------------------------------------------------------------------------------------------
# (2) library level: the mixer through the C ABI against the oracle
RMS_TOL, MAX_TOL = 1e-6, 1e-5            # relative to the reference's peak
NBUF, BUF_FRAMES = 61, 8192
SIZES = (1024, 1024, 37, 1000, 1024, 1024, 1024, 1024)


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


def _shelf(gain_hf):
    """A direct-path high shelf at 5 kHz (no low shelf): a filter whose output the fp32
    recurrence does not amplify, so the usual bound holds."""
    lp = np.zeros(5, dtype=np.float32)
    hp = np.zeros(5, dtype=np.float32)
    lib = mixlib.product()
    assert lib.biquad_coeffs(0, 5000.0 / 48000.0, gain_hf, 1.0, lp.ctypes.data) == 0
    assert lib.biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data) == 0
    return lp, hp


HRTF_VOICES_MAX = 1000


class _Scene:
    """`n` parked voices on a `cw`-channel dry bus, then the update script of run().  On the HRTF
    device the odd voices of the first 2*h are HRTF voices besides them, h = min(n, 1000): past
    about a thousand HRTF voices the HRTF path's own fp32 sums (partial rows per CTA against the
    oracle's one running sum) reach 1e-6 of the peak by themselves, whichever path the dry bus
    takes, and what is under test here is the dry bus."""

    def __init__(self, device, n):
        self.hrtf = device == "hrtf16"
        self.cw = 16 if self.hrtf else int(device[4:])
        self.nh = min(n, HRTF_VOICES_MAX) if self.hrtf else 0
        self.n0 = n + self.nh
        self.nadd = max(70, n // 8)                       # parked voices added later
        nv = self.n0 + self.nadd
        if self.hrtf:
            self.desc = synth.hrtf_desc(nv, 64, dry_channels=16)
        else:
            self.desc = synth.stereo_desc(nv, dry_channels=self.cw)
            self.desc.real_channels = self.cw
            self.desc.post_process = abi.POST_NONE
        self.desc.max_buffers = NBUF
        rng = np.random.default_rng(4000 + n + self.cw)
        self.params, self.coeffs, self.dry = synth.voice_set(
            rng, nv, 64 if self.hrtf else 0, hrtf=False, dry_channels=self.cw, frames=BUF_FRAMES)
        self.dry *= np.float32(scene.voice_gain(n) * 4.0)
        for k, p in enumerate(self.params):
            p.buffer = k % NBUF
            if self.is_hrtf(k):
                p.flags |= abi.VF_HRTF
            if k % 7 == 3:
                # one-shot, ending somewhere in the first updates (mid-update as a rule)
                p.flags &= ~abi.VF_LOOPING
                p.position = BUF_FRAMES - int(rng.integers(200, 6000))
        # (the one-shot voices are left alone by the later updates: they end on their own)
        rng2 = np.random.default_rng(99)
        self.moved = [k for k in range(self.n0) if k % 8 in (1, 2) and k % 7 != 3]
        self.moved_dry = (rng2.standard_normal((len(self.moved), self.cw)) * 0.3
                          * scene.voice_gain(n) * 4.0).astype(np.float32)
        self.stopped = [k for k in range(self.n0) if k % 11 == 5 and k % 7 != 3]
        self.lp, self.hp = _shelf(0.35)

    def is_hrtf(self, k):
        return k < 2 * self.nh and k % 2 == 1

    def _voices(self, idx, flags_set=0, flags_clear=0):
        out = []
        for k in idx:
            q = abi.VoiceParams.from_buffer_copy(bytes(self.params[k]))
            q.flags = (q.flags & ~flags_clear) | flags_set
            out.append(q)
        return out

    def _update(self, dev, idx, voices, dry=None):
        idx = np.asarray(idx)
        dev.voices_update(voices, self.coeffs[idx] if self.hrtf else None,
                          self.dry[idx] if dry is None else dry, None)

    def run(self, lib):
        """Returns ([(out, dry)] per update, product launch count or None)."""
        dev = MixDevice(lib, self.desc)
        if self.hrtf:
            dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7), 16))
        for b in range(NBUF):
            dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b, BUF_FRAMES))
        # 1. reset voices
        first = list(range(self.n0))
        self._update(dev, first, self._voices(first))
        res = []
        for u, f in enumerate(SIZES):
            if u == 1:
                # 2. new gains for a quarter, no reset: 64-sample fades in the first tile
                self._update(dev, self.moved, self._voices(self.moved, flags_clear=abi.VF_RESET),
                             self.moved_dry)
            if u == 4:
                # 4. direct filters on every third voice: their lines come from dline
                dev.voices_filters((k, 0, 1, self.lp, self.hp) for k in range(0, self.n0, 3))
            if u == 5:
                # 5. stop some voices (fade out this update)
                self._update(dev, self.stopped, self._voices(
                    self.stopped, flags_set=abi.VF_STOPPING, flags_clear=abi.VF_PLAYING | abi.VF_RESET))
            if u == 6:
                # ... then drop them, and 6. add voices: the entry list is rebuilt and crosses a
                # 64-entry chunk boundary
                self._update(dev, self.stopped, self._voices(
                    self.stopped, flags_set=abi.VF_STOPPED,
                    flags_clear=abi.VF_PLAYING | abi.VF_STOPPING | abi.VF_RESET))
                new = list(range(self.n0, self.n0 + self.nadd))
                self._update(dev, new, self._voices(new))
            out = dev.render(f)
            res.append((out, dev.dry()[:, :f]))
        launches = None
        if lib is mixlib.product():
            fn = lib.lib.b200mix_launch_count
            fn.restype, fn.argtypes = C.c_uint64, [C.c_void_p]
            launches = int(fn(dev.h))
        dev.close()
        return res, launches

    def parked_entries(self):
        """Parked entries of every update (the dry-bus entry list: active non-HRTF voices)."""
        parked = lambda ks: sum(1 for k in ks if not self.is_hrtf(k))  # noqa: E731
        before = parked(range(self.n0))
        after = before - parked(self.stopped) + parked(range(self.n0, self.n0 + self.nadd))
        return [before] * 6 + [after] * 2


def _check(got, ref, what):
    peak = max(float(np.abs(r).max()) for r in ref)
    assert peak > 1e-2, f"{what}: reference is silent"
    for u, (g, r) in enumerate(zip(got, ref)):
        err = g.astype(np.float64) - r.astype(np.float64)
        rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
        assert rms <= RMS_TOL * peak and mx <= MAX_TOL * peak, \
            f"{what}, update {u} ({SIZES[u]} frames): rms {rms:.3e} max {mx:.3e} peak {peak:.3e}"


@pytest.mark.parametrize("n", [65, 1000, 8200])
@pytest.mark.parametrize("device", ["none5", "none9", "none16", "hrtf16"])
def test_panmix_scene_vs_oracle(device, n):
    sc = _Scene(device, n)
    entries = sc.parked_entries()
    # every full update has more than one chunk of parked entries, so each one takes the tensor cores
    assert min(entries) > 64
    if n == 8200:
        assert any(chunking(e)[1][-1][0] == e for e in entries), "no empty trailing chunk"
    # the added voices move the entry count across a multiple of 64 entries
    assert (entries[-1] + 63) // 64 != (entries[0] + 63) // 64
    ref, _ = sc.run(mixlib.oracle())
    tc, launches_tc = sc.run(mixlib.product())
    with _env("B200MIX_PANMIX_SIMT", "1"):
        simt, launches_simt = sc.run(mixlib.product())
    for name, res in (("tensor cores", tc), ("SIMT", simt)):
        _check([dr for _, dr in res], [dr for _, dr in ref], f"{device} n={n} dry bus, {name}")
        _check([o for o, _ in res], [o for o, _ in ref], f"{device} n={n} output, {name}")
    # k_panmix_tc is the only launch the SIMT switch removes: it ran once per full update and on no
    # ragged one
    assert launches_tc - launches_simt == sum(f == LINE for f in SIZES), (launches_tc, launches_simt)
