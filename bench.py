#!/usr/bin/env python3
"""bench.py — the per-update mixing hot path on H100 (BASELINE.json metric:
"real-time HRTF voices @48kHz/1024-sample update; samples/sec mixed").

A step = ONE 1024-frame mix update of the whole voice set (the voice loop of
DeviceBase::renderSamples, alc/alu.cpp:2412) over synthetic 48 kHz mono voices.
N=1 workload = BASELINE config 2: 4096 mono voices, HRTF (64-tap HRIR pair per voice),
bsinc24, pitch in [0.5, 2.0) with 1/16 at 1.0 (SURVEY.md §8d).  N>1: 4096 voices per GPU
(weak scaling), a voice-sharded device set: the LIBRARY sums the ranks' RealOut blocks onto
rank 0 inside b200mix_render (peer stores over NVLink, or NCCL), and before anything is
printed rank 0 checks the reduced block of a 1/16 subsample against ONE device mixing those
same voices.

  python bench.py --gpus N --steps K --warmup W            # the CUDA mixer (libb200mix.so)
  python bench.py --impl reference --gpus N --steps K ...  # the reference's own CPU mixer
  python bench.py ... --dump-outputs DIR    # also writes the last timed update's RealOut block

value  : voice-samples/s with everything resident in HBM, device-timed (CUDA events on the
         mixer's stream around each update incl. the RealOut reduce, L2 flushed between
         updates; the K updates are enqueued back to back and the host synchronises once,
         after the last one), max over ranks.
e2e    : same metric through the C ABI with HOST buffers: per step the parameter snapshots of
         1/8 of the voices (moving sources) go host->device, the (reduced, on rank 0) planar
         output block and the per-voice results come back to host memory.
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "openal-soft_b200"))
from pyb200mix import abi, scene, shard  # noqa: E402

VOICES_PER_GPU = 4096
IR = 64
FRAMES = 1024
UPDATE_MS = 1000.0 * FRAMES / 48000.0
L2_FLUSH_BYTES = 256 << 20
WORKLOAD = ("config2: 4096 mono 48k voices per GPU, Default HRTF 64-tap HRIR pair per voice, "
            "bsinc24, pitch U[0.5,2) (1/16 at 1.0)")
METRIC = "voice-samples/s mixed (HRTF, bsinc24, 1024-frame updates)"
SUSTAINED_VOICES = 131072
FP32_LANES = 128                     # FP32 lanes per SM (Hopper)
HBM_GBS_DATASHEET = 3350.0           # H100 SXM data sheet


# --------------------------------------------------------------------------- helpers
def load_product():
    path = os.path.join(ROOT, "openal-soft_b200", "libb200mix.so")
    if not os.path.exists(path):
        raise SystemExit("libb200mix.so missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path)
    lib.b200mix_create.argtypes = [C.POINTER(abi.DeviceDesc), C.POINTER(C.c_void_p)]
    lib.b200mix_destroy.argtypes = [C.c_void_p]
    lib.b200mix_last_error.restype = C.c_char_p
    lib.b200mix_last_error.argtypes = [C.c_void_p]
    lib.b200mix_set_hrtf_decoder.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 3
    lib.b200mix_buffer_data.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.c_void_p, C.c_size_t]
    lib.b200mix_voices_update.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    lib.b200mix_render.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.c_void_p]
    lib.b200mix_render_device.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]
    lib.b200mix_profile.argtypes = [C.c_void_p, C.c_int]
    lib.b200mix_last_mix_kernel_ms.restype = C.c_float
    lib.b200mix_last_mix_kernel_ms.argtypes = [C.c_void_p]
    lib.b200mix_launch_count.restype = C.c_uint64
    lib.b200mix_launch_count.argtypes = [C.c_void_p]
    lib.b200mix_stream.restype = C.c_void_p
    lib.b200mix_stream.argtypes = [C.c_void_p]
    lib.b200mix_hrtf_load.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
    lib.b200mix_hrtf_get_coeffs.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
                                            C.c_void_p, C.POINTER(C.c_uint32)]
    lib.b200mix_hrtf_attach.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200mix_voices_update_dirs.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    lib.b200mix_shard_init.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.b200mix_shard_connect.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200mix_shard_nccl_id.argtypes = [C.c_void_p]
    lib.b200mix_shard_nccl.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.b200mix_shard_last_us.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lib.b200mix_resampler_taps.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    return lib


MHR_PATH = os.path.join(ROOT, "openal-soft_b200", "data", "Default HRTF.mhr")


def load_hrtf(lib):
    """The reference's default data set through the product's own MHR loader, or None."""
    if not os.path.exists(MHR_PATH):
        return None
    data = open(MHR_PATH, "rb").read()
    h = C.c_void_p()
    return h if lib.b200mix_hrtf_load(data, len(data), C.byref(h)) == 0 else None


def direction_of(pos):
    """{elevation, azimuth, distance, spread} as CalcHrtfPanning derives them for a source
    at `pos` (alc/alu.cpp:1210-1216)."""
    x, y, z = pos
    d = math.sqrt(x * x + y * y + z * z)
    ev = math.asin(max(-1.0, min(1.0, y / d)))
    az = math.atan2(x / d, -z / d)
    return ev, az, d, 0.0


def hrir_for(lib, hrtf, pos, out, delays):
    """HrtfStore::getCoeffs on the host for a source at `pos`."""
    ev, az, d, sp = direction_of(pos)
    lib.b200mix_hrtf_get_coeffs(hrtf, ev, az, d, sp, out.ctypes.data, delays)


def synth_voices(indices, total, lib=None, hrtf=None, shift=0.0):
    """Post-ALU parameter snapshots for the scene voices `indices` (global indices of a
    `total`-voice scene, SURVEY §8d positions) as local voices 0..n-1: HRIR pair + delays from
    Default HRTF.mhr via the product's HrtfStore::getCoeffs restatement (synthetic decaying
    filters only if the data set is not staged), gain 1/sqrt(total).  `shift` rotates the
    azimuths (moving sources)."""
    indices = list(indices)
    count = len(indices)
    rng = np.random.default_rng(0xB200 + (indices[0] if indices else 0))
    coeffs = (rng.standard_normal((count, IR, 2)) * np.exp(-np.arange(IR) / 10.0)[None, :, None]
              ).astype(np.float32)
    params = (abi.VoiceParams * max(count, 1))()
    dl = (C.c_uint32 * 2)()
    pitches = []
    cs, sn = math.cos(shift), math.sin(shift)
    for k, i in enumerate(indices):
        p = params[k]
        p.voice = k
        p.flags = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING | abi.VF_HRTF | abi.VF_RESET
        p.buffer = k
        p.resampler = abi.RS_BSINC24
        p.position = 0
        p.position_frac = 0
        p.loop_start = 0
        p.loop_end = scene.BUFFER_FRAMES
        pitch = scene.voice_pitch(i)
        pitches.append(pitch)
        p.step = max(1, min(int(pitch * 65536.0), 10 << 16))
        p.hrtf_delay[0] = int(rng.integers(0, 40))
        p.hrtf_delay[1] = int(rng.integers(0, 40))
        if hrtf is not None:
            x, y, z = scene.voice_position(i)
            if shift:
                x, z = x * cs - z * sn, x * sn + z * cs
            hrir_for(lib, hrtf, (x, y, z), coeffs[k], dl)
            p.hrtf_delay[0], p.hrtf_delay[1] = dl[0], dl[1]
        p.hrtf_gain = scene.voice_gain(total)
        for s in range(abi.MAX_SENDS):
            p.send_slot[s] = abi.NO_SLOT
    return params, coeffs, np.array(pitches)


def algorithmic_bytes_per_voice(mean_pitch):
    """SURVEY.md §8(d): source 1024*p*2 B + mPrevSamples R+W 2*192 + pos/frac/step 16
    + HRTF history R+W 2*256 + target coeffs Ir*8 + delays/gain 12."""
    return 1024.0 * mean_pitch * 2 + 2 * 192 + 16 + 2 * 256 + IR * 8 + 12


def algorithmic_flops(lib, h, params, count):
    """SURVEY.md §8(d) "algorithmic flops": per output sample FastBSinc 3m, BSinc 7m (0 for the
    pitch-1.0 copy), HRTF 4*Ir + 2."""
    total = 0.0
    full = C.c_uint32()
    for k in range(count):
        step = params[k].step
        m = lib.b200mix_resampler_taps(h, params[k].resampler, step, C.byref(full))
        rs = 0 if step == 65536 else (7 * m if full.value else 3 * m)
        total += FRAMES * (rs + 4 * IR + 2)
    return total


class ClockSampler:
    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.samples = []
        self.reasons = set()
        self.max_mhz = None
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits",
                                      "-i", str(self.idx)], capture_output=True, text=True, timeout=5).stdout
                f = [x.strip() for x in out.strip().split(",")]
                self.samples.append(float(f[0]))
                self.max_mhz = float(f[1])
                for n, v in zip(names, f[2:6]):
                    if v.lower().startswith("active"):
                        self.reasons.add(n)
            except Exception:
                pass
            self._stop.wait(0.2)

    def start(self):
        self._t.start()

    def stop(self):
        self._stop.set()
        self._t.join(timeout=6)
        med = float(np.median(self.samples)) if self.samples else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons)}


# --------------------------------------------------------------------------- reference arm
def physical_cpus():
    """One logical CPU per physical core among the CPUs this process may use."""
    allowed = sorted(os.sched_getaffinity(0))
    seen, out = set(), []
    for c in allowed:
        try:
            sib = open(f"/sys/devices/system/cpu/cpu{c}/topology/thread_siblings_list").read().strip()
        except OSError:
            sib = str(c)
        if sib not in seen:
            seen.add(sib)
            out.append(c)
    return out or allowed


def _ref_worker(first, count, total, steps, warmup, cpu, conn):
    if cpu is not None:
        try:
            os.sched_setaffinity(0, {cpu})
        except OSError:
            pass
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import refal
    dev = refal.RefDevice({refal.ALC_HRTF_SOFT: 1, refal.ALC_MONO_SOURCES: max(count, 1)})
    assert dev.hrtf_enabled()
    for k in range(count):
        i = first + k
        dev.add_voice(scene.voice_buffer_fast(i), scene.BUFFER_RATE, scene.voice_pitch(i),
                      scene.voice_position(i), scene.voice_gain(total), abi.RS_BSINC24)
    dev.play_all()
    for _ in range(warmup):
        dev.render()
    conn.send("ready")
    conn.recv()
    t0 = time.perf_counter()
    for _ in range(steps):
        dev.render()
    dt = time.perf_counter() - t0
    conn.send(dt)
    dev.close()


def run_reference(voices_per_proc, steps, warmup, cpus):
    """The reference's own SSE mixer (oracle/_ref/libopenal_ref.so through the loopback API):
    one independent loopback device per process, one process pinned to each CPU of `cpus`
    (the reference mixer is single-threaded per device, core/device.h:420-421), all released
    together.  Returns the per-process wall times of the timed `steps` updates."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    total = voices_per_proc * len(cpus)
    workers = []
    for r, cpu in enumerate(cpus):
        a, b = ctx.Pipe()
        pr = ctx.Process(target=_ref_worker, args=(r * voices_per_proc, voices_per_proc, total, steps,
                                                   warmup, cpu, b))
        pr.start()
        workers.append((pr, a))
    for _, a in workers:
        assert a.recv() == "ready"
    for _, a in workers:
        a.send("go")
    times = [a.recv() for _, a in workers]
    for pr, _ in workers:
        pr.join()
    return times


def reference_available():
    return (os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libopenal_ref.so"))
            and os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libref_harness.so")))


REF_US_PER_VOICE_UPDATE = 31.0       # the reference's SSE mixer, config-2 voices, one core (measured)


def main_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    if not reference_available():
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref not built"}))
        return
    cpus = physical_cpus()
    # A loaded sample: every process (one per physical core, pinned) mixes enough config-2
    # voices that the K timed updates take >= ~1.2 s — the reference's cost per voice-update is
    # constant, so its voice-samples/s on this sample IS its throughput on the config; a
    # sample of 4096 voices split over 64 cores would time 2 ms of work per step.
    per = int(math.ceil(1.2e6 / (max(args.steps, 1) * REF_US_PER_VOICE_UPDATE)))
    per = int(min(4096, max(512, ((per + 255) // 256) * 256)))
    times = run_reference(per, args.steps, args.warmup, cpus)
    sample = per * len(cpus)
    tmax, tmed = max(times), float(np.median(times))
    value = sample * FRAMES * args.steps / tmax
    line = {
        "impl": "reference", "metric": METRIC,
        "value": value, "unit": "voice-samples/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1000.0 * tmax / args.steps, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "voices_mixed": sample, "voices_per_process": per,
                   "update_frames": FRAMES},
        "cpu_baseline": {"value": value, "unit": "voice-samples/s", "cores": len(cpus), "kind": "reference",
                         "sample": f"{per} config-2 voices per process x {args.steps} updates, {len(cpus)} "
                                   f"independent loopback devices pinned one per physical core, SSE4.1 kernels",
                         "value_median_process": sample * FRAMES * args.steps / tmed,
                         "seconds_per_process": {"median": tmed, "max": tmax, "min": min(times)}},
        "e2e": {"value": value, "unit": "voice-samples/s", "h2d_bytes_per_step": 0,
                "d2h_bytes_per_step": 0},
        "rt_voices": sample * UPDATE_MS / (1000.0 * tmax / args.steps),
    }
    print(json.dumps(line))


# --------------------------------------------------------------------------- CUDA arm
def dump_real_out(torch, ptr, out_dir):
    """Copies the [2][1024] float RealOut block b200mix_render_device left at device address
    `ptr` to out_dir/real_out.npy (float32)."""
    class _Block:
        __cuda_array_interface__ = {"shape": (2, FRAMES), "typestr": "<f4", "data": (ptr, False),
                                    "strides": None, "version": 2}
    out = torch.as_tensor(_Block(), device="cuda").cpu().numpy()
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "real_out.npy"), out)


class Mixer:
    """One b200mix device holding the scene voices `indices` (global indices) as local voices."""

    def __init__(self, lib, local, indices, total, hrtf, pool=0):
        self.lib, self.indices, self.total = lib, list(indices), total
        nv = len(self.indices)
        desc = abi.DeviceDesc()
        desc.struct_size = C.sizeof(abi.DeviceDesc)
        desc.cuda_device = local
        desc.sample_rate = 48000
        desc.dry_channels = 4
        desc.real_channels = 2
        desc.ir_size = IR
        desc.post_process = abi.POST_HRTF
        desc.real_left, desc.real_right = 0, 1
        desc.max_voices = max(nv, 1)
        desc.max_buffers = max(nv, 1)
        self.h = C.c_void_p()
        rc = lib.b200mix_create(C.byref(desc), C.byref(self.h))
        if rc != 0:
            raise SystemExit(f"b200mix_create failed: {lib.b200mix_last_error(None)}")
        rng = np.random.default_rng(7)
        dec = (rng.standard_normal((4, 91, 2)) * np.exp(-np.arange(91) / 12.0)[None, :, None] * 0.2
               ).astype(np.float32)
        hf = np.array([2.0, 1.1547005, 1.1547005, 1.1547005], dtype=np.float32)
        sc = np.full(4, -0.9123257, dtype=np.float32)
        self.ck(lib.b200mix_set_hrtf_decoder(self.h, 4, 91, dec.ctypes.data, hf.ctypes.data, sc.ctypes.data),
                "set_hrtf_decoder")
        cache = {}
        for k, i in enumerate(self.indices):
            # every voice owns a PRIVATE device buffer (SURVEY §8d); with `pool` the host-side
            # waveform is taken from a pool of that many distinct signals (upload time only)
            key = i % pool if pool else i
            pcm = cache.get(key)
            if pcm is None:
                pcm = scene.voice_buffer_fast(key)
                if pool:
                    cache[key] = pcm
            self.ck(lib.b200mix_buffer_data(self.h, k, abi.FMT_I16, 1, pcm.shape[0], pcm.ctypes.data, pcm.nbytes),
                    "buffer_data")
        self.params, self.coeffs, self.pitches = synth_voices(self.indices, total, lib, hrtf)
        if nv:
            self.ck(lib.b200mix_voices_update(self.h, nv, self.params, self.coeffs.ctypes.data, None, None),
                    "voices_update")
        self.out_ptr = C.c_void_p()

    def ck(self, rc, what):
        if rc != 0:
            raise SystemExit(f"{what} failed ({rc}): {self.lib.b200mix_last_error(self.h)}")

    def render_device(self):
        self.ck(self.lib.b200mix_render_device(self.h, FRAMES, C.byref(self.out_ptr)), "render_device")

    def render_host(self, results=None):
        out = np.zeros((2, FRAMES), dtype=np.float32)
        ptrs = (C.c_void_p * 2)(out[0].ctypes.data, out[1].ctypes.data)
        self.ck(self.lib.b200mix_render(self.h, FRAMES, ptrs, results), "render")
        return out

    def close(self):
        if self.h:
            self.lib.b200mix_destroy(self.h)
            self.h = None


def connect_shard(mx, rank, world, transport, gloo):
    """Joins mx's device to the sharded set.  Handles / the NCCL id travel over the gloo
    group of torch.distributed — host plumbing; the exchange itself is the library's."""
    shard.connect(mx.lib, mx.h, rank, world, transport, gloo)


def verify_sharded(lib, local, rank, world, hrtf, gloo, transports):
    """Before any number is printed: a 1/16 subsample of the 4096*N voices is mixed (a) by the
    sharded set, every rank holding its own share, reduced by the library onto rank 0, and
    (b) by ONE device on rank 0 holding all of them; 4 updates must agree within
    north_star's tolerance (RMS 1e-5, max 1e-4 — in practice fp32 re-association, ~1e-7)."""
    import torch.distributed as dist
    total = VOICES_PER_GPU * world
    first = VOICES_PER_GPU * rank
    mine = [i for i in range(first, first + VOICES_PER_GPU) if i % 16 == 0]
    report = {}
    single = None
    if rank == 0:
        sx = Mixer(lib, local, [i for i in range(total) if i % 16 == 0], total, hrtf)
        single = np.stack([sx.render_host() for _ in range(4)])
        sx.close()
    for tr in transports:
        mx = Mixer(lib, local, mine, total, hrtf)
        connect_shard(mx, rank, world, tr, gloo)
        outs = np.stack([mx.render_host() for _ in range(4)])
        dist.barrier(group=gloo)
        mx.close()
        if rank == 0:
            err = outs.astype(np.float64) - single
            rms, mxe = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
            peak = float(np.abs(single).max())
            if not (peak > 1e-3 and rms <= 1e-5 and mxe <= 1e-4):
                raise SystemExit(f"bench.py: the {tr} reduce of {world} ranks does NOT equal the single-device "
                                 f"mix (rms {rms:.3e}, max {mxe:.3e}, peak {peak:.3e}) — no number printed")
            report[tr] = {"rms": rms, "max": mxe, "peak": peak}
    return {"voices": len(mine) * world, "updates": 4, "vs": "one device mixing the same voices", **report}


def main_cuda(args):
    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — the b200mix mixer has no CPU path")
    torch.cuda.set_device(local)
    gloo = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        gloo = dist.new_group(backend="gloo")
    lib = load_product()
    hrtf = load_hrtf(lib)

    total = VOICES_PER_GPU * world
    first = VOICES_PER_GPU * rank
    nv = VOICES_PER_GPU

    verification = None
    transports = ["p2p", "nccl"] if world > 1 else []
    if world > 1:
        verification = verify_sharded(lib, local, rank, world, hrtf, gloo, transports)

    mx = Mixer(lib, local, range(first, first + nv), total, hrtf)
    h = mx.h
    ck = mx.ck
    stream = torch.cuda.ExternalStream(lib.b200mix_stream(h))
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device="cuda")

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed_device_steps(steps, warmup, dump=None):
        """K device-timed updates: events on the mixer's stream around every update, L2 flushed
        before each, the K updates enqueued back to back and the host synchronised once at the end
        (the contract's bracket) — a per-update host round trip would put host wake-up jitter of
        the slowest of N processes into every rank-0 reduce.  A short host-synchronous pass
        afterwards samples the per-kernel / per-collective device times.
        With `dump` (rank 0), the RealOut block of the last timed update is written there.
        Returns (per-step ms, per-step voice-kernel ms, per-step reduce us, launches)."""
        for _ in range(warmup):
            mx.render_device()
        barrier()
        l0 = lib.b200mix_launch_count(h)
        evs = []
        for _ in range(steps):
            with torch.cuda.stream(stream):
                flush.zero_()                       # evict the voice state / sources from L2
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            mx.render_device()                      # incl. the library's RealOut reduce when sharded
            e1.record(stream)
            evs.append((e0, e1))
        torch.cuda.synchronize()
        launches = lib.b200mix_launch_count(h) - l0
        if dump and rank == 0:
            dump_real_out(torch, mx.out_ptr.value, dump)
        step_ms = [a.elapsed_time(b) for a, b in evs]
        mix_ms, red_us = [], []
        ru = C.c_float(-1.0)
        for _ in range(min(steps, 4)):
            with torch.cuda.stream(stream):
                flush.zero_()
            mx.render_device()
            torch.cuda.synchronize()
            mix_ms.append(lib.b200mix_last_mix_kernel_ms(h))
            if world > 1:
                lib.b200mix_shard_last_us(h, None, C.byref(ru))
                red_us.append(ru.value)
        barrier()
        return step_ms, mix_ms, red_us, launches

    def max_over_ranks(x):
        if world == 1:
            return x
        tt = torch.tensor([x], device="cuda", dtype=torch.float64)
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        return float(tt.item())

    # ---- device-timed value -------------------------------------------------------
    collective = None
    nccl_ms = None
    if world > 1:
        # the NCCL transport first (a quarter of the steps, for the comparison line), then the
        # peer-store transport the headline is measured on
        connect_shard(mx, rank, world, "nccl", gloo)
        lib.b200mix_profile(h, 1)
        s_ms, _, r_us, _ = timed_device_steps(max(4, args.steps // 4), args.warmup)
        nccl_ms = max_over_ranks(float(np.mean(s_ms)))
        nccl_red = max_over_ranks(float(np.mean(r_us)))
        connect_shard(mx, rank, world, "p2p", gloo)
    lib.b200mix_profile(h, 1)
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    step_ms, mix_ms, red_us, launches = timed_device_steps(args.steps, args.warmup, args.dump_outputs)
    lib.b200mix_profile(h, 0)
    alg_flops = algorithmic_flops(lib, h, mx.params, nv)
    t_total = max_over_ranks(float(np.sum(step_ms)))
    ms_per_step = t_total / args.steps
    value = total * FRAMES / (ms_per_step * 1e-3)
    if world > 1:
        collective = {"transport": "peer stores over NVLink (CUDA IPC), rank-ordered sum on rank 0",
                      "bytes": 2 * FRAMES * 4,
                      "reduce_us": max_over_ranks(float(np.mean(red_us))),
                      "reduce_us_note": "device time of the reduce on its stream in a host-synchronous pass (on rank 0 "
                                        "it includes waiting for the slowest rank's block), max over ranks",
                      "nccl": {"ms_per_step": nccl_ms, "reduce_us": nccl_red,
                               "what": "same update with ncclReduce (library transport 2)"}}

    # ---- end-to-end through the C ABI with host buffers ----------------------------
    results = (abi.VoiceResult * nv)()
    nmove = nv // 8
    h2d = nmove * (C.sizeof(abi.VoiceParams) + IR * 2 * 4)
    d2h = 2 * FRAMES * 4 + nv * C.sizeof(abi.VoiceResult)
    # the application's per-update work (new positions -> new HRIRs) is prepared up
    # front: 8 rotating sets, each moving a different eighth of the voices
    move_sets = []
    for base in range(8):
        idx = [first + base + 8 * j for j in range(nmove)]
        p2, c2, _ = synth_voices(idx, total, lib, hrtf, shift=0.05 * (base + 1))
        md = np.zeros((nmove, 4), dtype=np.float32)
        cs, sn = math.cos(0.05 * (base + 1)), math.sin(0.05 * (base + 1))
        for j in range(nmove):
            k = base + 8 * j
            p2[j].voice = k
            p2[j].buffer = k
            p2[j].flags &= ~abi.VF_RESET
            if hrtf is None:
                p2[j].hrtf_delay[0] = (mx.params[k].hrtf_delay[0] + 3 * base + 1) % 40
            x, y, z = scene.voice_position(first + k)
            md[j] = direction_of((x * cs - z * sn, y, x * sn + z * cs))
        move_sets.append((p2, np.ascontiguousarray(c2), md))

    # With the data set attached the application only sends the moved sources' DIRECTIONS
    # and the 4-HRIR blend runs on the GPU (b200mix_voices_update_dirs, SURVEY §8f #1);
    # otherwise it sends host-blended HRIRs.
    use_dirs = hrtf is not None and lib.b200mix_hrtf_attach(h, hrtf) == 0
    if use_dirs:
        h2d = nmove * (C.sizeof(abi.VoiceParams) + 16)
    out = np.zeros((2, FRAMES), dtype=np.float32)
    ptrs = (C.c_void_p * 2)(out[0].ctypes.data, out[1].ctypes.data)

    def step_e2e(it):
        mp, mc, md = move_sets[it % 8]
        if use_dirs:
            ck(lib.b200mix_voices_update_dirs(h, nmove, mp, md.ctypes.data, None, None), "voices_update_dirs")
        else:
            ck(lib.b200mix_voices_update(h, nmove, mp, mc.ctypes.data, None, None), "voices_update")
        # sharded: the render ends with the SUMMED block in rank 0's host buffer
        ck(lib.b200mix_render(h, FRAMES, ptrs, results), "render")

    for it in range(args.warmup):
        step_e2e(it)
    barrier()
    t0 = time.perf_counter()
    for it in range(args.steps):
        step_e2e(args.warmup + it)
    torch.cuda.synchronize()
    te = max_over_ranks(time.perf_counter() - t0)
    e2e_value = total * FRAMES * args.steps / te
    clk = clocks.stop() if rank == 0 else None

    sustained = None
    if world > 1:
        dist.barrier()          # nobody unmaps its receive block while a peer may still write to it
    mx.close()
    del flush
    if world == 1 and not args.no_sustained:
        sustained = run_sustained(lib, local, hrtf, torch)
    cpu = None
    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", HBM_GBS_DATASHEET))
        peak_src = ("MEASURED_PEAKS.json hbm_gbs (burst copy)" if peaks
                    else f"H100 SXM data sheet {HBM_GBS_DATASHEET:.0f} GB/s")
        mean_pitch = float(np.mean(mx.pitches))
        alg_bytes = algorithmic_bytes_per_voice(mean_pitch) * nv
        good = [m for m in mix_ms if m > 0]
        mix_avg = float(np.mean(good)) if good else None
        achieved = alg_bytes / (mix_avg * 1e-3) / 1e9 if mix_avg else None
        num_sms = torch.cuda.get_device_properties(local).multi_processor_count
        sm_max = float((clk or {}).get("sm_max_mhz") or peaks.get("sm_max_mhz", 1980.0))
        fp32_peak = num_sms * FP32_LANES * 2 * sm_max * 1e6 / 1e12           # TFLOP/s
        fp32_ach = alg_flops / (mix_avg * 1e-3) / 1e12 if (mix_avg and alg_flops) else None
        fracs = {"hbm": (achieved / peak) if achieved else None,
                 "fp32": (fp32_ach / fp32_peak) if fp32_ach else None}
        bound = max((k for k in fracs if fracs[k] is not None), key=lambda k: fracs[k], default="hbm")
        line = {
            "metric": METRIC,
            "value": value, "unit": "voice-samples/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD,
                       "voices": total, "voices_per_gpu": nv, "update_frames": FRAMES,
                       "hrir": ("Default HRTF.mhr (MinPHR03, 48 kHz, Ir=64) via b200mix_hrtf_get_coeffs"
                                if hrtf is not None else "synthetic decaying 64-tap pairs (data set not staged)"),
                       "l2": "flushed between timed updates (256 MiB memset)",
                       "parallelism": (f"voices sharded over {world} GPU(s); the library reduces RealOut onto "
                                       f"rank 0 inside b200mix_render (peer stores over NVLink)")},
            "rt_voices": total * UPDATE_MS / ms_per_step,
            "e2e": {"value": e2e_value, "unit": "voice-samples/s", "h2d_bytes_per_step": h2d * world,
                    "d2h_bytes_per_step": d2h * world, "ms_per_step": 1000.0 * te / args.steps,
                    "update": ("b200mix_voices_update_dirs (directions; HRIR blend on the GPU)" if use_dirs
                               else "b200mix_voices_update (host-blended HRIRs)")
                              + f", {nmove} moved voices/GPU/update"
                              + ("; the RealOut reduce is inside b200mix_render and rank 0's host buffer "
                                 "receives the summed block" if world > 1 else "")},
            "gpu_launches": int(launches),
            "gpu": torch.cuda.get_device_name(local),
            "clocks": clk,
            "roofline": {"bound": bound, "kernel": "k_mix_voices",
                         "achieved": achieved, "peak": peak, "unit": "GB/s",
                         "frac": fracs["hbm"],
                         "peak_source": peak_src,
                         "kernel_ms": mix_avg, "algorithmic_bytes_per_launch": alg_bytes,
                         "fp32": {"achieved": fp32_ach, "peak": fp32_peak, "unit": "TFLOP/s", "frac": fracs["fp32"],
                                  "algorithmic_flops_per_launch": alg_flops,
                                  "peak_source": f"{num_sms} SMs x {FP32_LANES} lanes x 2 x {sm_max:.0f} MHz"},
                         "note": "frac is the algorithmic-bytes/HBM figure; an HRTF voice is ~100 flop/B, "
                                 "so the kernel is bounded by shared-memory traffic and FP32 issue, not by "
                                 "HBM — `bound` names the higher of the two fractions"},
        }
        if collective:
            line["collective"] = collective
        if verification:
            line["verification"] = verification
        if sustained:
            line["sustained"] = sustained
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline()
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_sustained(lib, local, hrtf, torch):
    """131 072 voices (one GPU's share of config 5's million), each on a PRIVATE 48 000-frame
    buffer (12.6 GB — far beyond L2, so no flush is needed), mixed back to back for >= 2 s with
    the SM clock sampled: rt_voices measured under sustained load instead of extrapolated."""
    nv = SUSTAINED_VOICES
    t0 = time.perf_counter()
    mx = Mixer(lib, local, range(nv), nv, hrtf, pool=512)
    setup_s = time.perf_counter() - t0
    stream = torch.cuda.ExternalStream(lib.b200mix_stream(mx.h))
    for _ in range(4):
        mx.render_device()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    mx.render_device()
    e1.record(stream)
    e1.synchronize()
    one = e0.elapsed_time(e1)
    updates = int(max(64, math.ceil(2200.0 / max(one, 1e-3))))
    clocks = ClockSampler(local)
    clocks.start()
    e0.record(stream)
    for _ in range(updates):
        mx.render_device()
    e1.record(stream)
    e1.synchronize()
    ms = e0.elapsed_time(e1)
    clk = clocks.stop()
    mx.close()
    per = ms / updates
    return {"voices": nv, "updates": updates, "seconds": ms / 1000.0, "ms_per_update": per,
            "value": nv * FRAMES / (per * 1e-3), "unit": "voice-samples/s",
            "rt_voices": nv * UPDATE_MS / per, "clocks": clk,
            "buffers": f"{nv} private 48000-frame i16 buffers ({nv * 96000 / 1e9:.1f} GB)",
            "setup_seconds": setup_s}


def cpu_baseline():
    """The reference's SSE mixer on ONE host core (it is single-threaded per device by
    design), bounded sample: 1024 config-2 voices x 32 updates (~1 s)."""
    if not reference_available():
        return {"value": None, "unit": "voice-samples/s", "cores": 1, "kind": "reference",
                "sample": "unavailable: oracle/_ref not built"}
    sample, steps = 1024, 32
    dt = run_reference(sample, steps, 4, physical_cpus()[:1])[0]
    return {"value": sample * FRAMES * steps / dt, "unit": "voice-samples/s", "cores": 1,
            "kind": "reference",
            "sample": f"{sample} config-2 voices x {steps} updates, 1 loopback device pinned to one core, "
                      f"SSE4.1 kernels",
            "ms_per_voice_update": 1000.0 * dt / (sample * steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-sustained", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed update's RealOut block as DIR/real_out.npy (float32)")
    args = ap.parse_args()
    if args.impl == "reference":
        main_reference(args)
    else:
        main_cuda(args)


if __name__ == "__main__":
    main()
