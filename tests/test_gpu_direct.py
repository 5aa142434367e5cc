"""Direct-channel voices (b200mix_voices_update_direct, AL_DIRECT_CHANNELS_SOFT) on the GPU.

A direct voice's line goes into RealOut ahead of the post-process, so on every post kind that
takes them RealOut is (direct sum) + post-process output.  The oracle has no direct path of its
own; the expected output is composed from two oracle devices that see the same voices:
  - the scene's device, where each direct voice mixes into Dry with zero gains (it still runs
    through the resampler, feeds nothing and leaves the post-process as it was), and
  - a device without a post-process whose Dry mix has RealOut's channels, where each direct voice
    mixes with its RealOut gains and its direct filter — which is the reference's Mix_ of the
    voice into RealOut (Dry is RealOut there).
BS2B's cross-feed runs on the decode only and the direct L/R are added back after it, so the
same composition holds with BS2B installed."""
import ctypes as C

import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

VF_DIRECT = 1 << 8
ERR_INVALID, ERR_UNSUPPORTED = -1, -4
RMS_TOL, MAX_TOL = 1e-6, 1e-5


def _lib():
    lib = mixlib.product().lib
    f = lib.b200mix_voices_update_direct
    f.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.b200mix_launch_count.argtypes = [C.c_void_p]
    lib.b200mix_launch_count.restype = C.c_uint64
    return lib


def _direct(dev, params, real, send=None, expect=0):
    n = len(params)
    arr = (abi.VoiceParams * n)(*params)
    real = None if real is None else np.ascontiguousarray(real, dtype=np.float32)
    rc = _lib().b200mix_voices_update_direct(dev.h, n, arr, None if real is None else real.ctypes.data,
                                             None if send is None else send.ctypes.data)
    assert rc == expect, (rc, dev.last_error())


def _launches(dev):
    return int(_lib().b200mix_launch_count(dev.h))


def _copy(p, flags=None):
    q = abi.VoiceParams()
    C.memmove(C.byref(q), C.byref(p), C.sizeof(p))
    if flags is not None:
        q.flags = flags
    return q


def _shelf_pair(gain_hf, gain_lf):
    lp = np.zeros(5, dtype=np.float32)
    hp = np.zeros(5, dtype=np.float32)
    lib = mixlib.product()
    assert lib.biquad_coeffs(0, 5000.0 / 48000.0, gain_hf, 1.0, lp.ctypes.data) == 0
    assert lib.biquad_coeffs(1, 250.0 / 48000.0, gain_lf, 1.0, hp.ctypes.data) == 0
    return lp, hp


KINDS = ["hrtf", "stereo", "stereo_bs2b", "surround51", "surround51_dual"]
CONV_IR = (np.random.default_rng(9).standard_normal((1, 300)) * np.exp(-np.arange(300) / 75.0) * 0.05
           ).astype(np.float32)


def _device_desc(kind, nv):
    if kind == "hrtf":
        return synth.hrtf_desc(nv, 64)
    if kind.startswith("stereo"):
        return synth.stereo_desc(nv, 3)           # <= 4 dry channels: the register-dry k_mix_voices
    if kind == "wide71":
        d = synth.stereo_desc(nv, 3)              # 7.1 from a first-order 2D mix: RealOut rows are
        d.real_channels = 8                       # wider than Dry's
        return d
    d = synth.stereo_desc(nv, 9)                  # second-order dry mix: the parking k_mix_voices
    d.real_channels = 6
    return d


def _setup_post(dev, kind):
    desc = dev.desc
    if kind == "hrtf":
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        return
    rng = np.random.default_rng(3)
    hf = (rng.standard_normal((desc.dry_channels, desc.real_channels)) * 0.5).astype(np.float32)
    lf = (rng.standard_normal((desc.dry_channels, desc.real_channels)) * 0.5).astype(np.float32)
    dev.set_ambi_decoder(hf, lf if kind.endswith("dual") else None, -0.9)
    if kind == "stereo_bs2b":
        dev.set_bs2b(4)
    if desc.max_slots:
        dev.slot_convolution(0, CONV_IR, np.full((1, desc.dry_channels), 0.5, np.float32))


def _aux_desc(desc):
    d = synth.stereo_desc(desc.max_voices, desc.real_channels)
    d.post_process = abi.POST_NONE
    d.real_channels = desc.real_channels
    return d


class Scene:
    """nn normal voices (HRTF on the HRTF device) and nd direct voices after them, a script of
    updates between renders: real-gain changes (fades), a direct filter, a stop, a removal.
    `sends`: every second voice also feeds a convolution slot through one aux send; `oneshot`:
    the second direct voice does not loop and runs out of samples within the scene."""

    def __init__(self, kind, nn, nd, seed=11, sends=False, oneshot=False):
        rng = np.random.default_rng(seed)
        self.kind, self.nn, self.nd = kind, nn, nd
        nv = nn + nd
        self.desc = _device_desc(kind, nv)
        if sends:
            self.desc.num_sends, self.desc.wet_channels, self.desc.max_slots = 1, 4, 1
        hrtf = kind == "hrtf"
        ir = self.desc.ir_size
        self.params, self.coeffs, self.dry = synth.voice_set(rng, nv, ir, hrtf=hrtf,
                                                             dry_channels=self.desc.dry_channels)
        for p in self.params[nn:]:
            p.flags &= ~abi.VF_HRTF
        self.send = None
        if sends:
            self.send = (rng.standard_normal((nv, 1, 4)) * 0.3).astype(np.float32)
            for k, p in enumerate(self.params):
                p.send_slot[0] = 0 if k % 2 else abi.NO_SLOT
        if oneshot and nd > 1:
            p = self.params[nn + 1]
            p.flags &= ~abi.VF_LOOPING
            p.position = scene.BUFFER_FRAMES - 600
        R = self.desc.real_channels
        self.real = [(rng.standard_normal((nd, R)) * 0.3).astype(np.float32) for _ in range(3)]
        self.filt = _shelf_pair(0.3, 0.7)
        self.pcm = [scene.voice_buffer_fast(i) for i in range(nv)]

    def load(self, dev, first=0):
        for i in range(first, self.nn + self.nd):
            dev.buffer_data(i, abi.FMT_I16, self.pcm[i])

    def direct_params(self, update):
        """The direct voices' entries of update 0, 1 or 2 (flags without VF_DIRECT)."""
        out = []
        for k, p in enumerate(self.params[self.nn:]):
            if update == 0:
                out.append(_copy(p))
                continue
            fl = p.flags & ~(abi.VF_RESET | abi.VF_FADING)
            if update == 2 and k == 0:
                fl = (fl & ~abi.VF_PLAYING) | abi.VF_STOPPING
            out.append(_copy(p, fl))
        return out

    def filters(self):
        lp, hp = self.filt
        return [(self.nn + k, 0, 1, lp, hp) for k in range(1, self.nd, 3)]

    def sends(self, direct):
        if self.send is None:
            return None
        return np.ascontiguousarray(self.send[self.nn:] if direct else self.send[:self.nn])

    def start_normal(self, dev):
        nn = self.nn
        if nn:
            dev.voices_update(self.params[:nn], self.coeffs[:nn] if self.desc.ir_size else None,
                              self.dry[:nn], self.sends(False))

    def run_product(self, sizes):
        dev = MixDevice(mixlib.product(), self.desc)
        _setup_post(dev, self.kind)
        self.load(dev)
        self.start_normal(dev)
        out, res = [], []
        for u, f in enumerate(sizes):
            if u < 3:
                dp = self.direct_params(u)
                for p in dp:
                    p.flags |= VF_DIRECT
                _direct(dev, dp, self.real[u], self.sends(True))
            if u == 1:
                dev.voices_filters(self.filters())
            o, r = dev.render(f, want_results=True)
            out.append(o)
            res.append([(x.position, x.position_frac, x.flags, x.buffers_done) for x in r])
        dev.close()
        return np.concatenate(out, axis=1), res

    def run_oracle(self, sizes):
        lib = mixlib.oracle()
        main, aux = MixDevice(lib, self.desc), MixDevice(lib, _aux_desc(self.desc))
        _setup_post(main, self.kind)
        self.load(main)
        self.load(aux, self.nn)
        nd = self.nd
        self.start_normal(main)
        zeros = np.zeros((nd, self.desc.dry_channels), dtype=np.float32)
        out, res = [], []
        for u, f in enumerate(sizes):
            if u < 3:
                main.voices_update(self.direct_params(u), None, zeros, self.sends(True))
                dp = self.direct_params(u)
                for p in dp:                      # the sends are the scene device's
                    p.send_slot[0] = abi.NO_SLOT
                aux.voices_update(dp, None, self.real[u])
            if u == 1:
                aux.voices_filters(self.filters())
            o, r = main.render(f, want_results=True)
            out.append(o.astype(np.float64) + aux.render(f).astype(np.float64))
            res.append([(x.position, x.position_frac, x.flags, x.buffers_done) for x in r])
        main.close()
        aux.close()
        return np.concatenate(out, axis=1), res


def _check(out, ref, what, rms_tol=RMS_TOL, max_tol=MAX_TOL):
    err = out.astype(np.float64) - ref
    rms = float(np.sqrt((err ** 2).mean()))
    mx = float(np.abs(err).max())
    assert rms <= rms_tol and mx <= max_tol, f"{what}: rms {rms:.3e} max {mx:.3e}"
    assert np.abs(ref).max() > 1e-4, "reference output is silent"


SIZES = {"full": (1024, 1024, 1024, 1024), "ragged": (333, 1, 1024, 17, 700)}


@pytest.mark.parametrize("sizes", list(SIZES))
@pytest.mark.parametrize("kind", KINDS)
def test_direct_voices_vs_oracle(kind, sizes):
    sc = Scene(kind, nn=24, nd=8)
    got, gres = sc.run_product(SIZES[sizes])
    ref, rres = sc.run_oracle(SIZES[sizes])
    assert gres == rres
    _check(got, ref, f"{kind} {sizes}")


@pytest.mark.parametrize("sizes", list(SIZES))
@pytest.mark.parametrize("kind", ["hrtf", "stereo", "surround51"])
def test_direct_voices_with_sends_and_a_oneshot_vs_oracle(kind, sizes):
    """Direct voices that also feed a convolution slot (their lines parked for both the sends and
    the RealOut bus), and one that runs out of samples and stops on its own."""
    sc = Scene(kind, nn=24, nd=8, seed=21, sends=True, oneshot=True)
    got, gres = sc.run_product(SIZES[sizes])
    ref, rres = sc.run_oracle(SIZES[sizes])
    assert gres == rres
    assert gres[-1][sc.nn + 1][2] == abi.VF_STOPPED          # the one-shot has ended
    _check(got, ref, f"{kind} {sizes} sends + one-shot")


def test_a_full_stage_of_direct_voices_on_a_device_with_more_real_than_dry_channels():
    """7.1 output from a 3-channel dry mix, 256 voices (the update arena's size at creation) all
    direct in one call: each carries 8 RealOut gains, more than the 3 dry gains a voice has."""
    sc = Scene("wide71", nn=0, nd=256, seed=31)
    # gains scaled by 1/sqrt(voices), as synth scales the other scenes' voices, so that the absolute
    # tolerance bounds the fp32 re-association of 256 lines as it does elsewhere (a gain row read
    # from the wrong place is off by ~0.1)
    sc.real = [r / 16.0 for r in sc.real]
    got, gres = sc.run_product((1024, 500, 1024))
    ref, rres = sc.run_oracle((1024, 500, 1024))
    assert gres == rres
    _check(got, ref, "256 direct voices, 8 RealOut channels")


def test_many_hrtf_voices_with_64_direct():
    sc = Scene("hrtf", nn=4096, nd=64, seed=5)
    got, gres = sc.run_product((1024, 1024))
    ref, rres = sc.run_oracle((1024, 1024))
    assert gres == rres
    # the HRIR FIR sums of 4096 voices are re-associated against the oracle's serial sum: DESIGN §4
    # measures 1.9e-6 / 1.6e-5 for 1200 HRTF voices, and that error grows with the square root of
    # the voice count (2.5e-6 / 1.7e-5 measured here on an H100); a wrong direct bus is off by the
    # direct voices' level, ~0.1
    _check(got, ref, "4096 HRTF + 64 direct", rms_tol=4e-6, max_tol=4e-5)


@pytest.mark.parametrize("kind", KINDS)
def test_device_whose_direct_voices_left_renders_as_one_that_never_had_any(kind):
    """Once its direct voices have left, a device launches the same kernels as a device with the
    same other voices that never had any, and renders the same RealOut.  Not bit for bit: in the
    update the direct voices still played, the other voices were spread over a grid sized for
    more voices, an fp32 re-association that the HRTF carry and BS2B's recurrences pass on."""
    sc = Scene(kind, nn=24, nd=4)
    nn = sc.nn
    counts, outs = [], []
    for with_direct in (False, True):
        dev = MixDevice(mixlib.product(), sc.desc)
        _setup_post(dev, kind)
        sc.load(dev)
        dev.voices_update(sc.params[:nn], sc.coeffs[:nn] if sc.desc.ir_size else None, sc.dry[:nn])
        dp = sc.direct_params(0)
        for p in dp:
            p.flags |= VF_DIRECT
        if with_direct:
            _direct(dev, dp, sc.real[0])
        dev.render(512)
        if with_direct:
            for p in dp:
                p.flags = abi.VF_STOPPED | VF_DIRECT
            _direct(dev, dp, None)
        c0 = _launches(dev)
        outs.append(np.concatenate([dev.render(f) for f in (1024, 77, 1024)], axis=1))
        counts.append(_launches(dev) - c0)
        dev.close()
    assert counts[0] == counts[1]
    _check(outs[1], outs[0].astype(np.float64), f"{kind} after the direct voices left")


@pytest.mark.parametrize("kind", KINDS)
def test_refused_batch_on_a_device_with_direct_voices_changes_nothing(kind):
    """A direct update whose last entry is refused (VF_HRTF) applies none of its entries, on a
    device whose RealOut bus is already live: it renders bit-identical to its twin without the
    call, with the same launches."""
    sc = Scene(kind, nn=24, nd=4)
    outs, counts = [], []
    for refused in (False, True):
        dev = MixDevice(mixlib.product(), sc.desc)
        _setup_post(dev, kind)
        sc.load(dev)
        sc.start_normal(dev)
        dp = sc.direct_params(0)
        for p in dp:
            p.flags |= VF_DIRECT
        _direct(dev, dp, sc.real[0])
        dev.render(512)
        if refused:
            bad = sc.direct_params(1)
            for p in bad:
                p.flags |= VF_DIRECT
            bad[-1].flags |= abi.VF_HRTF
            _direct(dev, bad, sc.real[1], expect=ERR_INVALID)
        c0 = _launches(dev)
        outs.append(np.concatenate([dev.render(f) for f in (1024, 300, 1024)], axis=1))
        counts.append(_launches(dev) - c0)
        dev.close()
    assert counts[0] == counts[1]
    assert outs[0].tobytes() == outs[1].tobytes()
    assert np.abs(outs[0]).max() > 1e-4


def _refusal_case(desc, setup, entries_flags, expect):
    """The refused call changes nothing: the device renders what its twin without the call does."""
    outs = []
    for call in (False, True):
        dev = MixDevice(mixlib.product(), desc)
        setup(dev)
        for i in range(4):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        params, _, dry = synth.voice_set(np.random.default_rng(1), 4, 0, hrtf=False,
                                         dry_channels=desc.dry_channels)
        dev.voices_update(params[:2], None, dry[:2])
        if call:
            dp = [_copy(p, (p.flags & ~abi.VF_HRTF) | entries_flags) for p in params[2:]]
            _direct(dev, dp, np.full((2, desc.real_channels), 0.5, np.float32), expect=expect)
        outs.append(np.concatenate([dev.render(f) for f in (1024, 100)], axis=1))
        dev.close()
    assert outs[0].tobytes() == outs[1].tobytes()
    assert np.abs(outs[0]).max() > 1e-4


def test_refusals_change_nothing():
    stereo = synth.stereo_desc(8, 3)

    def ambi(dev):
        _setup_post(dev, "stereo")
    # no VF_DIRECT, or VF_HRTF with it
    _refusal_case(stereo, ambi, 0, ERR_INVALID)
    _refusal_case(stereo, ambi, VF_DIRECT | abi.VF_HRTF, ERR_INVALID)
    # RealOut is the Dry mix
    none = synth.stereo_desc(8, 2)
    none.post_process = abi.POST_NONE
    _refusal_case(none, lambda dev: None, VF_DIRECT, ERR_UNSUPPORTED)
    # UHJ: the reference's RemixMap is empty
    uhj = synth.stereo_desc(8, 3)
    uhj.post_process = abi.POST_UHJ
    _refusal_case(uhj, lambda dev: dev.set_uhj_encoder(0), VF_DIRECT, ERR_UNSUPPORTED)
    # a front stabilizer
    s51 = _device_desc("surround51", 8)

    def stab(dev):
        _setup_post(dev, "surround51")
        dev.set_front_stabilizer(2, -0.9)
    _refusal_case(s51, stab, VF_DIRECT, ERR_UNSUPPORTED)


def test_stabilizer_refused_while_direct_voices_play():
    desc = _device_desc("surround51", 4)
    dev = MixDevice(mixlib.product(), desc)
    _setup_post(dev, "surround51")
    dev.buffer_data(0, abi.FMT_I16, scene.voice_buffer_fast(0))
    params, _, _ = synth.voice_set(np.random.default_rng(1), 1, 0, hrtf=False, dry_channels=9)
    params[0].flags |= VF_DIRECT
    _direct(dev, params, np.full((1, 6), 0.5, np.float32))
    assert dev.m.set_front_stabilizer(dev.h, 2, -0.9) == ERR_UNSUPPORTED
    params[0].flags = abi.VF_STOPPED | VF_DIRECT
    _direct(dev, params, None)
    dev.set_front_stabilizer(2, -0.9)
    dev.close()


def test_toggle_between_dry_and_direct_while_playing():
    """A voice moved from Dry to RealOut and back while it plays, on a device whose decode passes
    Dry channel c to RealOut channel c: with its gains unchanged the moves are inaudible, since
    the voice keeps one set of Current gains (the reference's mDryParams.Gains.Current)."""
    desc = synth.stereo_desc(4, 2)
    desc.real_channels = 2
    outs = []
    for toggle in (False, True):
        dev = MixDevice(mixlib.product(), desc)
        dev.set_ambi_decoder(np.eye(2, dtype=np.float32), None, 0.0)
        dev.buffer_data(0, abi.FMT_I16, scene.voice_buffer_fast(0))
        params, _, _ = synth.voice_set(np.random.default_rng(4), 1, 0, hrtf=False, dry_channels=2)
        g0 = np.array([[0.5, 0.25]], np.float32)
        g1 = np.array([[0.125, 0.75]], np.float32)
        dev.voices_update(params, None, g0)
        o = [dev.render(1024)]
        run = _copy(params[0], params[0].flags & ~(abi.VF_RESET | abi.VF_FADING))
        # a gain change that fades (the voice is fading from its second update on), then moves
        if toggle:
            _direct(dev, [_copy(run, run.flags | VF_DIRECT)], g1)
        else:
            dev.voices_update([run], None, g1)
        o.append(dev.render(1024))
        if toggle:
            dev.voices_update([run], None, g1)
        o.append(dev.render(1024))
        outs.append(np.concatenate(o, axis=1))
        dev.close()
    # the same gains reach the same channels; only the summation into RealOut differs (decode
    # of a one-hot matrix vs the RealOut bus): exact
    _check(outs[1], outs[0].astype(np.float64), "toggle")


def test_voice_moved_from_dry_to_realout_fades_from_its_dry_gains_vs_oracle():
    """The reference's voice keeps one mDryParams.Gains.Current whichever buffer it feeds: a voice
    moved from Dry to RealOut while it plays fades from the Current gains it had at the shared
    channel indices to its RealOut targets.  Expected: the voice on an oracle device without a
    post-process and RealOut's channels, with its Dry gains there first (that update's output not
    used), then its RealOut gains; plus the scene's device, where the voice leaves after the
    first update."""
    rng = np.random.default_rng(77)
    desc = synth.stereo_desc(8, 3)
    nn, v = 6, 6
    params, _, dry = synth.voice_set(rng, nn + 1, 0, hrtf=False, dry_channels=3)
    g0 = np.array([[0.6, -0.3, 0.4]], np.float32)
    r1 = np.array([[-0.2, 0.7]], np.float32)
    run = _copy(params[v], params[v].flags & ~(abi.VF_RESET | abi.VF_FADING))
    sizes = (1024, 700, 1024)
    pcm = [scene.voice_buffer_fast(i) for i in range(nn + 1)]

    dev = MixDevice(mixlib.product(), desc)
    _setup_post(dev, "stereo")
    for i in range(nn + 1):
        dev.buffer_data(i, abi.FMT_I16, pcm[i])
    dev.voices_update(params[:nn], None, dry[:nn])
    dev.voices_update([params[v]], None, g0)
    got = [dev.render(sizes[0])]
    _direct(dev, [_copy(run, run.flags | VF_DIRECT)], r1)
    got += [dev.render(f) for f in sizes[1:]]
    dev.close()

    lib = mixlib.oracle()
    main, aux = MixDevice(lib, desc), MixDevice(lib, _aux_desc(desc))
    _setup_post(main, "stereo")
    for i in range(nn + 1):
        main.buffer_data(i, abi.FMT_I16, pcm[i])
    aux.buffer_data(v, abi.FMT_I16, pcm[v])
    main.voices_update(params[:nn], None, dry[:nn])
    main.voices_update([params[v]], None, g0)
    aux.voices_update([params[v]], None, g0[:, :2])
    ref = [main.render(sizes[0]).astype(np.float64)]
    aux.render(sizes[0])
    main.voices_update([_copy(run, abi.VF_STOPPED)], None, None)
    aux.voices_update([run], None, r1)
    ref += [main.render(f).astype(np.float64) + aux.render(f) for f in sizes[1:]]
    main.close()
    aux.close()
    _check(np.concatenate(got, axis=1), np.concatenate(ref, axis=1), "Dry -> RealOut move")
