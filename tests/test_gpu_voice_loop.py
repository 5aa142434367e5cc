"""Every bus of the voice loop in the same updates, on one device that parks its dry bus.

A third-order ambisonic-decode device (16 dry channels, decoded to 6) runs, update after update:
  - more than 64 parked dry voices, so a full update's dry bus takes the tensor-core pan-mix;
  - direct-channel voices on the RealOut bus;
  - two convolution slots, each fed by more than 128 send entries, with send filters;
  - direct filters on some dry and some direct voices, so the filtered lines feed both buses;
  - voices that move between Dry, RealOut and stopped from one update to the next;
at full and ragged update sizes, one update through render_begin / render_end.

The oracle has no direct path of its own, so the expected RealOut is composed as in
test_gpu_direct.py: the scene's device, where a direct voice mixes into Dry with zero gains (and
feeds its sends), plus a device without a post-process whose Dry mix has RealOut's channels, where
it mixes with its RealOut gains and direct filter.  A voice that moves restarts (VF_RESET), so its
gains do not fade across the move on either side."""
import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene
from test_gpu_direct import VF_DIRECT, _aux_desc, _copy, _direct, _shelf_pair

pytestmark = pytest.mark.gpu

CD, REAL, CW = 16, 6, 4
NDRY, NDIRECT, NMOVE = 160, 24, 60              # static dry, static direct, moving voices
NV = NDRY + NDIRECT + NMOVE
NBUF, BUF_FRAMES = 61, 8192
SIZES = (1024, 1024, 333, 1024, 1, 1024, 700, 1024)
BEGIN = 5                                       # the update taken through render_begin / render_end
RMS_TOL, MAX_TOL = 1e-6, 1e-5                   # relative to the reference's peak (test_gpu_panmix)
DRY, DIRECT, STOPPED = 0, 1, 2


def _state(k, u):
    """Voice k's path in update u."""
    if k < NDRY:
        return DRY
    if k < NDRY + NDIRECT:
        return DIRECT
    return (k + u) % 3


class _Scene:
    def __init__(self):
        rng = np.random.default_rng(2024)
        self.desc = synth.stereo_desc(NV, CD)
        self.desc.real_channels = REAL
        self.desc.max_buffers = NBUF
        self.desc.num_sends, self.desc.wet_channels, self.desc.max_slots = 2, CW, 2
        self.params, _, dry = synth.voice_set(rng, NV, 0, hrtf=False, dry_channels=CD, frames=BUF_FRAMES)
        g = np.float32(scene.voice_gain(NV) * 4.0)
        self.dry = dry * g
        self.real = (rng.standard_normal((NV, REAL)) * 0.3 * g).astype(np.float32)
        self.send = (rng.standard_normal((NV, 2, CW)) * 0.3 * g).astype(np.float32)
        for k, p in enumerate(self.params):
            p.buffer = k % NBUF
            p.send_slot[0], p.send_slot[1] = 0, 1
        self.irs = [(rng.standard_normal((1, n)) * np.exp(-np.arange(n) / 75.0) * 0.05).astype(np.float32)
                    for n in (300, 700)]
        dec = np.random.default_rng(3)
        self.decode = (dec.standard_normal((CD, REAL)) * 0.3).astype(np.float32)
        self.shelf = _shelf_pair(0.3, 0.7)
        self.send_shelf = _shelf_pair(0.5, 0.8)

    def setup(self, dev):
        dev.set_ambi_decoder(self.decode, None, 0.0)
        for s, ir in enumerate(self.irs):
            dev.slot_convolution(s, ir, np.full((1, CD), 0.5, np.float32))
        for b in range(NBUF):
            dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b, BUF_FRAMES))

    def changed(self, u):
        """The voices whose path update u sets: all of them first, then the moving ones."""
        return list(range(NV)) if u == 0 else list(range(NDRY + NDIRECT, NV))

    def entry(self, k, u, state):
        p = self.params[k]
        if state == STOPPED:
            return _copy(p, abi.VF_STOPPED)
        return _copy(p, p.flags | abi.VF_RESET) if u == 0 or k >= NDRY + NDIRECT else _copy(p)

    def filters(self, direct_only):
        """Direct filters on every fourth dry and every third direct voice; send filters (product
        and the scene's oracle device) on every fifth voice's first send and every seventh's second."""
        lp, hp = self.shelf
        out = [(k, 0, 1, lp, hp) for k in range(NDRY, NDRY + NDIRECT, 3)]
        if direct_only:
            return out
        slp, shp = self.send_shelf
        out += [(k, 0, 1, lp, hp) for k in range(0, NDRY, 4)]
        out += [(k, 1, 1, slp, shp) for k in range(0, NV, 5)]
        return out + [(k, 2, 1, slp, shp) for k in range(0, NV, 7)]

    def parked(self, u):
        """Entries of the dry bus and of each slot in update u."""
        st = [_state(k, u) for k in range(NV)]
        return st.count(DRY), NV - st.count(STOPPED)

    def run_product(self):
        dev = MixDevice(mixlib.product(), self.desc)
        self.setup(dev)
        out = []
        for u, f in enumerate(SIZES):
            ks = self.changed(u)
            by = {s: [k for k in ks if _state(k, u) == s] for s in (DRY, DIRECT, STOPPED)}
            if by[DRY]:
                dev.voices_update([self.entry(k, u, DRY) for k in by[DRY]], None, self.dry[by[DRY]],
                                  self.send[by[DRY]])
            if by[DIRECT]:
                dp = [self.entry(k, u, DIRECT) for k in by[DIRECT]]
                for p in dp:
                    p.flags |= VF_DIRECT
                _direct(dev, dp, self.real[by[DIRECT]], np.ascontiguousarray(self.send[by[DIRECT]]))
            if by[STOPPED]:
                dev.voices_update([self.entry(k, u, STOPPED) for k in by[STOPPED]])
            if u == 0:
                dev.voices_filters(self.filters(False))
            if u == BEGIN:
                dev.render_begin(f)
                out.append(dev.render_end())
            else:
                out.append(dev.render(f))
        dev.close()
        return out

    def run_oracle(self):
        lib = mixlib.oracle()
        main, aux = MixDevice(lib, self.desc), MixDevice(lib, _aux_desc(self.desc))
        self.setup(main)
        for b in range(NBUF):
            aux.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b, BUF_FRAMES))
        out = []
        for u, f in enumerate(SIZES):
            ks = self.changed(u)
            st = [_state(k, u) for k in ks]
            main.voices_update([self.entry(k, u, s) for k, s in zip(ks, st)], None,
                               np.where(np.array(st)[:, None] == DRY, self.dry[ks], 0.0), self.send[ks])
            ap = []
            for k, s in zip(ks, st):
                p = self.entry(k, u, s if s == DIRECT else STOPPED)
                p.send_slot[0] = p.send_slot[1] = abi.NO_SLOT
                ap.append(p)
            aux.voices_update(ap, None, self.real[ks])
            if u == 0:
                main.voices_filters(self.filters(False))
                aux.voices_filters(self.filters(True))
            out.append(main.render(f).astype(np.float64) + aux.render(f))
        main.close()
        aux.close()
        return out


def test_every_bus_in_the_same_updates_vs_oracle():
    sc = _Scene()
    for u, f in enumerate(SIZES):
        dry, slot = sc.parked(u)
        if f == 1024:
            assert dry > 64, "the full updates' dry bus takes the tensor cores"
        assert slot > 128, "each slot's sends take more than one entry chunk"
    ref = sc.run_oracle()
    got = sc.run_product()
    peak = max(float(np.abs(r).max()) for r in ref)
    assert peak > 1e-2, "reference is silent"
    for u, (g, r) in enumerate(zip(got, ref)):
        err = g.astype(np.float64) - r
        rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
        assert rms <= RMS_TOL * peak and mx <= MAX_TOL * peak, \
            f"update {u} ({SIZES[u]} frames): rms {rms:.3e} max {mx:.3e} peak {peak:.3e}"
