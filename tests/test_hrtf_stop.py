"""Stopping HRTF voices against a float64 restatement of DoHrtfMix, at every HRIR length.

A voice that stops (VF_STOPPING, or a one-shot that ran out) fades out over one update:
DoHrtfMix (core/voice.cpp:827-902) blends its old HRIR down to silence and mixes nothing new.
These scenes put every such case next to playing voices:
  - stopped by an update with no new parameters, with new HRIRs (the old HRIR is mixed),
    with new delays only and with a new gain only;
  - stopped on the update right after a reset, with and without VF_FADING on the reset;
  - a one-shot that runs out during an update, fades on the next and is then stopped;
  - a one-shot that ran out and is then given new parameters with VF_PLAYING (no reset): with
    no buffer it mixes its held last sample for one update, then stops like any voice that has
    none (core/voice.cpp:1224-1232);
  - a stopping voice with a zero step (it stops without mixing);
  - the updates after a stop, where the stopped voice leaves only its carried tail.

Every buffer is float32 and every step is 65536 with a zero fraction, so the line each voice
mixes is its buffer's samples (the resampler's copy path); every voice but a few silent dry
ones is an HRTF voice, so RealOut is the HRTF accumulator plus the tail it carries.  The
reference below restates DoHrtfMix, MixHrtfBlendBase and MixHrtfBase (hrtfbase.h:17-89) in
float64: the gains and gain steps are float32 in the reference's operation order (they decide
branches), the products and sums are float64.  Each output sample must be within a few float32
epsilons of the sum of the magnitudes of the terms that make it up.

Without a GPU this holds the CPU oracle to the restatement; with one (-m gpu) it holds the
CUDA mixer to both, and its voice positions and states to the oracle's exactly.  The GPU
scenes also mix stopping voices through a direct filter, against the oracle only."""
import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi

EPS32 = float(np.finfo(np.float32).eps)
K_F64 = 8.0                # per-sample bound: K_F64 * eps32 * sum |coef * x * gain|
SILENCE = np.float32(0.00001)      # GainSilenceThreshold, core/mixer/defs.h:28
HIST = abi.HRTF_HISTORY
FRAMES = 4096
NBUF = 64
IRS = [8, 9, 40, 63, 64, 65, 72, 100, 127, 128]
SIZES = [1, 3, 63, 64, 65, 517, 1024]
NROLES = 14
(PLAY, PLAY2, PLAY_NEWHRIR, STOP, STOP_HRIR, STOP_DELAY, STOP_GAIN, RESET_FADE_STOP,
 RESET_STOP, ONESHOT, STEP0, PLAY3, DRY, ONESHOT_UPDATED) = range(NROLES)
FILTER_ROLES = (PLAY, STOP, STOP_HRIR, STOP_GAIN)
RESAMPLERS = [abi.RS_POINT, abi.RS_LINEAR, abi.RS_BSINC24, abi.RS_FAST_BSINC12]
f32 = np.float32


def _copy(p):
    return abi.VoiceParams.from_buffer_copy(bytes(p))


def _scene(nv, ir, n, seed, filtered=False, roles=None):
    """The call sequence: a list of ("update", params, coeffs or None), ("filters", entries)
    and ("render",) steps, plus the buffers.  Renders 0..4 are updates U0..U4.  roles: voice
    k's role (default: k % NROLES).  filtered: a direct filter on some voices of FILTER_ROLES;
    "only": those voices are the only audible ones."""
    rng = np.random.default_rng(seed)
    bufs = rng.uniform(-1.0, 1.0, (NBUF, FRAMES)).astype(np.float32)
    params, coeffs, _ = synth.voice_set(rng, nv, ir, frames=FRAMES)
    dry = np.zeros((nv, 4), dtype=np.float32)
    roles = roles or [k % NROLES for k in range(nv)]
    for k, p in enumerate(params):
        p.buffer = k % NBUF
        p.resampler = RESAMPLERS[k % len(RESAMPLERS)]
        p.step, p.position_frac = 65536, 0
        p.position = int(rng.integers(0, FRAMES))
        if roles[k] in (ONESHOT, ONESHOT_UPDATED):      # runs out during U1
            p.flags &= ~abi.VF_LOOPING
            p.position = FRAMES - n - int(rng.integers(1, n + 1))
        if roles[k] == DRY:                     # a silent dry voice the HRIR FIR skips
            p.flags &= ~abi.VF_HRTF
    steps = [("update", [_copy(p) for p in params], coeffs.copy(), dry)]
    if filtered:
        lp = np.zeros(5, dtype=np.float32)
        hp = np.zeros(5, dtype=np.float32)
        ora = mixlib.oracle()
        assert ora.biquad_coeffs(0, 5000.0 / 48000.0, 0.35, 1.0, lp.ctypes.data) == 0
        assert ora.biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data) == 0
        chosen = [k for k in range(nv) if roles[k] in FILTER_ROLES and k % 2 == 0]
        steps.append(("filters", [(k, 0, 1, lp, hp) for k in chosen]))
        if filtered == "only":
            # the other voices are still mixed, with silent HRIRs: the sum is the filtered
            # voices' alone, so its float32 rounding stays small next to the bound
            silent = np.ones(nv, dtype=bool)
            silent[chosen] = False
            coeffs[silent] = 0.0
            steps[0] = ("update", steps[0][1], coeffs.copy(), dry)
    steps.append(("render",))

    def upd(ks, change, with_coeffs):
        if not ks:
            return
        out = []
        for k in ks:
            q = _copy(params[k])
            q.flags &= ~(abi.VF_RESET | abi.VF_FADING)
            change(k, q)
            params[k] = q
            out.append(_copy(q))
        steps.append(("update", out, coeffs[ks].copy() if with_coeffs else None, dry[ks]))

    def of(*rs):
        return [k for k in range(nv) if roles[k] in rs]

    def stopping(k, q):
        q.flags = (q.flags & ~abi.VF_PLAYING) | abi.VF_STOPPING

    def restart(fading):
        def change(k, q):
            q.flags |= abi.VF_RESET | (abi.VF_FADING if fading else 0)
            q.position = int(rng.integers(0, FRAMES))
        return change

    # U1: stops in every form, restarts, new HRIRs on playing voices
    coeffs[of(STOP_HRIR, PLAY_NEWHRIR)] = coeffs[of(STOP_HRIR, PLAY_NEWHRIR)][:, ::-1, :] * 0.6
    coeffs[of(RESET_FADE_STOP, RESET_STOP)] *= -0.8

    def stop_hrir(k, q):
        stopping(k, q)
        q.hrtf_delay[0] = (q.hrtf_delay[0] + 5) % HIST
        q.hrtf_gain *= 0.7

    def new_hrir(k, q):
        q.hrtf_delay[1] = (q.hrtf_delay[1] + 9) % HIST

    def stop_delay(k, q):
        stopping(k, q)
        q.hrtf_delay[1] = (q.hrtf_delay[1] + 7) % HIST

    def stop_gain(k, q):
        stopping(k, q)
        q.hrtf_gain *= 1.3

    def step0(k, q):
        stopping(k, q)
        q.step = 0

    upd(of(STOP), stopping, False)
    upd(of(STOP_HRIR), stop_hrir, True)
    upd(of(STOP_DELAY), stop_delay, False)
    upd(of(STOP_GAIN), stop_gain, False)
    upd(of(STEP0), step0, False)
    upd(of(PLAY_NEWHRIR), new_hrir, True)
    upd([k for k in of(RESET_FADE_STOP)], restart(True), True)
    upd([k for k in of(RESET_STOP)], restart(False), True)
    steps.append(("render",))
    # U2: the restarted voices stop; the one-shots fade out, or play on without a buffer
    upd(of(RESET_FADE_STOP, RESET_STOP), stopping, False)

    def replay(k, q):
        q.hrtf_delay[0] = (q.hrtf_delay[0] + 3) % HIST
        q.hrtf_gain *= 1.1

    upd(of(ONESHOT_UPDATED), replay, False)
    steps.append(("render",))
    # U3: the faded one-shots are stopped; U4: tails only for everything stopped
    upd(of(ONESHOT), lambda k, q: setattr(q, "flags", (q.flags & ~abi.VF_PLAYING) | abi.VF_STOPPED),
        False)
    steps.append(("render",))
    steps.append(("render",))
    return bufs, steps


def _play(lib, nv, ir, n, bufs, steps):
    """Runs the steps on one implementation; returns [(out, results)] per render."""
    desc = synth.hrtf_desc(nv, ir)
    desc.max_buffers = NBUF
    dev = MixDevice(lib, desc)
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7), ir=ir))
    for b in range(NBUF):
        dev.buffer_data(b, abi.FMT_F32, bufs[b])
    outs = []
    for st in steps:
        if st[0] == "update":
            dev.voices_update(st[1], st[2], st[3], None)
        elif st[0] == "filters":
            dev.voices_filters(st[1])
        else:
            out, res = dev.render(n, want_results=True)
            outs.append((out, [(r.position, r.position_frac, r.flags) for r in res[:nv]]))
    dev.close()
    return outs


class _Voice:
    pass


def _reference(nv, ir, n, bufs, steps):
    """float64 DoHrtfMix over the same steps: [(out, magnitude, results)] per render, where
    magnitude[c][i] = sum of |coef * x * gain| over the terms of out[c][i]."""
    vs = [None] * nv
    acc = np.zeros((2, n + abi.HRIR_LENGTH))
    mag = np.zeros((2, n + abi.HRIR_LENGTH))
    renders = []

    def add(coef, x, g, at):
        """accum[at + i + j] += coef[j] * x[i] * g[i] for both ears."""
        if len(g) == 0:
            return
        for e in range(2):
            term = x[e] * g.astype(np.float64)
            c = coef[:, e].astype(np.float64)
            acc[e, at:at + len(g) + ir - 1] += np.convolve(term, c)
            mag[e, at:at + len(g) + ir - 1] += np.convolve(np.abs(term), np.abs(c))

    def update(params, coeffs):
        for i, p in enumerate(params):
            if not p.flags & abi.VF_HRTF:
                continue
            v = vs[p.voice]
            if p.flags & abi.VF_RESET:               # Voice::prepare + InitVoice
                v = vs[p.voice] = _Voice()
                v.hist = np.zeros(HIST)
                v.tgt_coef = np.zeros((ir, 2), np.float32)
                v.old_coef = np.zeros((ir, 2), np.float32)
                v.old_delay, v.old_gain = (0, 0), f32(0.0)
                v.pos, v.frac, v.have_buffer = p.position, p.position_frac, True
                v.fading = bool(p.flags & abi.VF_FADING)
            if p.flags & abi.VF_STOPPED:
                v.state = 0
            elif p.flags & abi.VF_STOPPING:
                v.state = 2
            elif p.flags & abi.VF_PLAYING:
                v.state = 1
            v.looping = bool(p.flags & abi.VF_LOOPING)
            v.buf, v.step = p.buffer, p.step
            v.loop_start, v.loop_end = p.loop_start, p.loop_end
            v.tgt_delay = (int(p.hrtf_delay[0]), int(p.hrtf_delay[1]))
            v.tgt_gain = f32(p.hrtf_gain)
            if coeffs is not None:
                v.tgt_coef = coeffs[i].copy()

    def line(v):
        b = bufs[v.buf].astype(np.float64)
        if not v.have_buffer:
            # ended: the resampler holds the sample nearest 0 of the padding kept from the last
            # update, all of it the buffer's last sample here (core/voice.cpp:704-719)
            return np.full(n, b[-1])
        p = v.pos + np.arange(n)
        if v.looping:
            ls, le = v.loop_start, v.loop_end
            p = np.where(p >= le, (p - ls) % (le - ls) + ls, p)
            return b[p]
        return b[np.minimum(p, FRAMES - 1)]

    def mix(v):
        if v.state not in (1, 2):
            return
        if v.step < 1:                      # nothing to mix; a stopping voice stops
            if v.state == 2:
                v.state = 0
            return
        assert v.step == 65536 and v.frac == 0
        x = line(v)
        counter = min(n, 64) if v.fading else 0
        if not counter:
            v.old_coef, v.old_delay, v.old_gain = v.tgt_coef, v.tgt_delay, v.tgt_gain
        playing = v.state == 1
        target = f32(v.tgt_gain * f32(1.0 if playing else 0.0))
        hs = np.concatenate([v.hist, x])
        if playing:
            v.hist = hs[n:n + HIST].copy()

        def ears(delay, start, count):
            return [hs[HIST - delay[e] + start:HIST - delay[e] + start + count] for e in range(2)]

        fademix = 0
        if counter:
            # MixHrtfBlendBase over fademix = counter samples (counter <= n, so no lerp)
            fademix = min(n, counter)
            gain = target
            new_step = f32(gain / f32(fademix))
            old_step = f32(v.old_gain / f32(fademix))
            if v.old_gain > SILENCE:
                g = old_step * (fademix - np.arange(fademix)).astype(np.float32)
                add(v.old_coef, ears(v.old_delay, 0, fademix), g, 0)
            if f32(new_step * f32(fademix)) > SILENCE:
                g = new_step * np.arange(1, fademix).astype(np.float32)
                add(v.tgt_coef, ears(v.tgt_delay, 1, fademix - 1), g, 1)
            v.old_coef, v.old_delay, v.old_gain = v.tgt_coef, v.tgt_delay, gain
        if fademix < n:
            # MixHrtfBase: the steady ramp from Old.Gain to the target
            todo = n - fademix
            step = f32(f32(target - v.old_gain) / f32(todo))
            g = (v.old_gain + step * np.arange(todo).astype(np.float32)).astype(np.float32)
            add(v.tgt_coef, ears(v.tgt_delay, fademix, todo), g, fademix)
            v.old_gain = target
        v.fading = True
        if v.state == 2:
            v.state = 0
            return
        v.pos += n
        if v.have_buffer:
            if v.looping:
                if v.pos >= v.loop_end:
                    v.pos = (v.pos - v.loop_start) % (v.loop_end - v.loop_start) + v.loop_start
            elif v.pos >= FRAMES:
                v.have_buffer = False
        if not v.have_buffer:
            v.state = 2                     # Stopping: fades out on the next update

    for st in steps:
        if st[0] == "update":
            update(st[1], st[2])
        elif st[0] == "render":
            for v in vs:
                if v is not None:
                    mix(v)
            res = {k: (v.pos, v.frac, abi.VF_PLAYING if v.state == 1 else
                       abi.VF_STOPPING if v.state == 2 else abi.VF_STOPPED)
                   for k, v in enumerate(vs) if v is not None}
            renders.append((acc[:, :n].copy(), mag[:, :n].copy(), res))
            # the accumulator's tail moves to the front (alc/alu.cpp ProcessHrtf)
            for a in (acc, mag):
                a[:, :abi.HRIR_LENGTH] = a[:, n:n + abi.HRIR_LENGTH].copy()
                a[:, abi.HRIR_LENGTH:] = 0.0
    return renders


def _check_vs_reference(got, ref, what, k=K_F64):
    worst = 0.0
    for u, ((out, res), (r_out, r_mag, r_res)) in enumerate(zip(got, ref)):
        err = np.abs(out.astype(np.float64) - r_out)
        bound = k * EPS32 * r_mag
        bad = err > bound
        assert not bad.any(), (
            f"{what} update {u}: {int(bad.sum())} samples outside the bound, worst "
            f"{float(err.max()):.3e} ({float((err / np.maximum(r_mag, 1e-30)).max()) / EPS32:.1f} eps "
            f"of the term sum) at {np.unravel_index(int(np.argmax(err - bound)), err.shape)}")
        worst = max(worst, float((err / np.maximum(r_mag, 1e-30)).max()) / EPS32)
        for v, want in r_res.items():
            assert res[v] == want, f"{what} update {u} voice {v}: {res[v]} != {want}"
    return worst


def _peak_rel(got, ref):
    """Worst |got - ref| over the run, relative to the run's peak (for reports)."""
    a = np.concatenate([o for o, _ in got], axis=1).astype(np.float64)
    b = np.concatenate([o for o, _ in ref], axis=1).astype(np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


CPU_CASES = [(40, ir, n) for ir in IRS for n in SIZES] + [(3000, 40, 1024), (3000, 128, 517)]


@pytest.mark.parametrize("nv,ir,n", CPU_CASES)
def test_oracle_vs_float64(nv, ir, n):
    bufs, steps = _scene(nv, ir, n, seed=nv + 131 * ir + n)
    ref = _reference(nv, ir, n, bufs, steps)
    # (a 1-frame update can be silent: the first samples mix the zeroed histories)
    assert max(float(np.abs(r[0]).max()) for r in ref) > 0.0, "the run is silent"
    _check_vs_reference(_play(mixlib.oracle(), nv, ir, n, bufs, steps), ref, f"oracle nv {nv} ir {ir} n {n}")


GPU_CASES = ([(40, ir, n) for ir in IRS for n in SIZES]
             + [(3000, ir, n) for ir in IRS for n in (3, 65)]
             + [(3000, ir, 1024) for ir in (40, 64, 128)])


@pytest.mark.gpu
@pytest.mark.parametrize("nv,ir,n", GPU_CASES)
def test_kernel_vs_float64_and_oracle(nv, ir, n):
    bufs, steps = _scene(nv, ir, n, seed=nv + 131 * ir + n)
    ref = _reference(nv, ir, n, bufs, steps)
    got = _play(mixlib.product(), nv, ir, n, bufs, steps)
    ora = _play(mixlib.oracle(), nv, ir, n, bufs, steps)
    _check_vs_reference(got, ref, f"kernel nv {nv} ir {ir} n {n}")
    for u, ((o, res), (r, rres)) in enumerate(zip(got, ora)):
        err = np.abs(o.astype(np.float64) - r.astype(np.float64))
        bound = 2.0 * K_F64 * EPS32 * ref[u][1]
        assert (err <= bound).all(), f"kernel vs oracle update {u}: worst {float(err.max()):.3e}"
        assert res == rres, f"update {u}: voice results differ from the oracle's"


@pytest.mark.gpu
@pytest.mark.parametrize("ir", IRS)
@pytest.mark.parametrize("nv,n,filtered", [(40, 517, True), (40, 63, True), (3000, 1024, "only")])
def test_kernel_vs_oracle_filtered(nv, ir, n, filtered):
    """Stopping voices whose line comes through an active direct filter (the filtered line
    that k_hrtf_fir mixes), against the oracle.  The run is checked as one block against its
    peak (the bounds of tests/test_gpu_fir_stage.py): the filtered lines have no float64
    restatement here to bound each sample by.  With 3000 voices only the filtered ones are
    audible."""
    bufs, steps = _scene(nv, ir, n, seed=7 * nv + ir + n, filtered=filtered)
    got = _play(mixlib.product(), nv, ir, n, bufs, steps)
    ora = _play(mixlib.oracle(), nv, ir, n, bufs, steps)
    for u, ((_, res), (_, rres)) in enumerate(zip(got, ora)):
        assert res == rres, f"update {u}: voice results differ from the oracle's"
    o = np.concatenate([x for x, _ in got], axis=1).astype(np.float64)
    r = np.concatenate([x for x, _ in ora], axis=1).astype(np.float64)
    peak = float(np.abs(r).max())
    assert peak > 1e-4, "reference output is silent"
    err = np.abs(o - r) / peak
    rms, mx = float(np.sqrt((err ** 2).mean())), float(err.max())
    assert rms <= 1e-6 and mx <= 1e-5, f"nv {nv} ir {ir} n {n}: rms {rms:.3e} max {mx:.3e}"
