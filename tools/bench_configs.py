#!/usr/bin/env python3
"""Secondary measurement (NOT the driver's bench line — that is bench.py on config 2):
device-timed update cost of every BASELINE.json config shape on N GPUs.

    python tools/bench_configs.py --config 3                      # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \\
        --master-port 29511 tools/bench_configs.py --config 5 --gpus 8

Configs (BASELINE.json `configs`, SURVEY.md §8d); voices are sharded by index across ranks:
  1   64 voices, stereo (pairwise first-order dry mix + BFormatDec 3->2), spline
  2   4096 HRTF voices, bsinc24                                   (bench.py's workload)
  3   16384 HRTF voices + 32 EAX reverb slots
  4a  65536 voices into a third-order B-Format output (16 dry channels, no post-process)
  4b  65536 voices, 2-D first order + UHJ encode
  5   1M HRTF voices + 128 convolution (96000-tap IR) + 128 reverb slots
With --gpus N>1 the ranks form a sharded device set (b200mix_shard_*): slots are owned by rank
(slot mod N) and b200mix_render_device itself reduce-scatters the wet buffers and reduces
RealOut onto rank 0 (--transport p2p: peer stores over NVLink; nccl: ncclAllReduce + ncclReduce).
--voices overrides the TOTAL voice count (a single GPU can run its 1/N share of config 4/5
with --voices and --slot-share).  --filters adds an active direct low-pass to every voice.
Time: CUDA events on the mixer's stream around the whole update, L2 flushed between
updates, max over ranks.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "openal-soft_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
from pyb200mix import abi, scene, shard  # noqa: E402

CONFIGS = {
    "1": dict(voices=64, kind="stereo", resampler=abi.RS_SPLINE, conv=0, reverb=0),
    "2": dict(voices=4096, kind="hrtf", resampler=abi.RS_BSINC24, conv=0, reverb=0),
    "3": dict(voices=16384, kind="hrtf", resampler=abi.RS_BSINC24, conv=0, reverb=32),
    "4a": dict(voices=65536, kind="ambi3", resampler=abi.RS_BSINC24, conv=0, reverb=0),
    "4b": dict(voices=65536, kind="uhj", resampler=abi.RS_BSINC24, conv=0, reverb=0),
    "5": dict(voices=1 << 20, kind="hrtf", resampler=abi.RS_BSINC24, conv=128, reverb=128),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3", choices=sorted(CONFIGS))
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--voices", type=int, default=0, help="override the total voice count")
    ap.add_argument("--slot-share", type=int, default=1,
                    help="install only every k-th slot (one GPU standing for 1/k of the box)")
    ap.add_argument("--taps", type=int, default=96000)
    ap.add_argument("--filters", action="store_true")
    ap.add_argument("--pcm-pool", type=int, default=0,
                    help="distinct PCM contents (0 = one per voice up to 8192 voices per rank, else 256); "
                         "every voice still owns its own device buffer")
    ap.add_argument("--transport", default="p2p", choices=["p2p", "nccl"])
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed update's RealOut block as DIR/real_out_<config>.npy (float32)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    cfg = dict(CONFIGS[args.config])
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"launch with torchrun --nproc-per-node {args.gpus}"
    torch.cuda.set_device(local)
    gloo = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        gloo = dist.new_group(backend="gloo")
    total = args.voices or cfg["voices"]
    first, nv = shard.shard_range(total, world, rank)
    nslots = cfg["conv"] + cfg["reverb"]

    lib = bench.load_product()
    lib.b200mix_slot_reverb.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.ReverbParams)]
    lib.b200mix_slot_convolution.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.b200mix_slot_output_gains.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.b200mix_render_begin.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    lib.b200mix_render_end.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.b200mix_voices_filters.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    lib.b200mix_biquad_coeffs.argtypes = [C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_void_p]
    lib.b200mix_set_ambi_decoder.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_float]

    kind = cfg["kind"]
    desc = abi.DeviceDesc()
    desc.struct_size = C.sizeof(abi.DeviceDesc)
    desc.cuda_device = local
    desc.sample_rate = 48000
    desc.max_voices = desc.max_buffers = max(nv, 1)
    desc.real_left, desc.real_right = 0, 1
    if kind == "hrtf":
        desc.dry_channels, desc.real_channels, desc.ir_size = 4, 2, 64
        desc.post_process = abi.POST_HRTF
    elif kind == "stereo":
        desc.dry_channels, desc.real_channels, desc.ir_size = 3, 2, 0
        desc.post_process = abi.POST_AMBIDEC
    elif kind == "ambi3":
        desc.dry_channels, desc.real_channels, desc.ir_size = 16, 16, 0
        desc.post_process = abi.POST_NONE
    else:
        desc.dry_channels, desc.real_channels, desc.ir_size = 3, 2, 0
        desc.post_process = abi.POST_UHJ
    if nslots:
        desc.num_sends, desc.wet_channels, desc.max_slots = 1, 4, nslots
    h = C.c_void_p()
    assert lib.b200mix_create(C.byref(desc), C.byref(h)) == 0, lib.b200mix_last_error(None)
    rng = np.random.default_rng(7)
    if kind == "hrtf":
        dec = (rng.standard_normal((4, 91, 2)) * 0.05).astype(np.float32)
        hf = np.array([2.0, 1.1547005, 1.1547005, 1.1547005], dtype=np.float32)
        sc = np.full(4, -0.9123257, dtype=np.float32)
        lib.b200mix_set_hrtf_decoder(h, 4, 91, dec.ctypes.data, hf.ctypes.data, sc.ctypes.data)
    elif kind == "stereo":
        g = (rng.standard_normal((3, 2)) * 0.5).astype(np.float32)
        assert lib.b200mix_set_ambi_decoder(h, 3, g.ctypes.data, None, 0.0) == 0

    # ---- effect slots: convolution first, then reverb; a rank installs the slots it owns ----
    installed = 0
    if nslots:
        fx = dict(np.load(os.path.join(ROOT, "tests", "golden", "hrtf_bsinc24_reverb_v6.npz")))
        rp = abi.reverb_params_from(fx["reverb_params"].tobytes())
        rp.struct_size = C.sizeof(abi.ReverbParams)
        rg = np.ascontiguousarray(fx["reverb_gains"], dtype=np.float32)
        for s in range(nslots):
            if shard.slot_owner(s, world) != rank or (s // world) % args.slot_share:
                continue
            if s < cfg["conv"]:
                ir = (np.random.default_rng(0xC0FFEE ^ s).standard_normal((1, args.taps))
                      * np.exp(-np.arange(args.taps) / (args.taps / 6.0)) * 0.02).astype(np.float32)
                g = np.array([[0.5, 0.0, 0.0, 0.8]], dtype=np.float32)
                assert lib.b200mix_slot_convolution(h, s, 1, args.taps, ir.ctypes.data) == 0, \
                    lib.b200mix_last_error(h)
                lib.b200mix_slot_output_gains(h, s, 1, g.ctypes.data)
            else:
                assert lib.b200mix_slot_reverb(h, s, C.byref(rp)) == 0, lib.b200mix_last_error(h)
                lib.b200mix_slot_output_gains(h, s, 8, rg.ctypes.data)
            installed += 1

    # ---- voices ----
    hrtf = bench.load_hrtf(lib) if kind == "hrtf" else None
    pool = args.pcm_pool or (nv if nv <= 8192 else 256)
    pcms = {}
    for k in range(nv):
        key = (first + k) % pool
        if key not in pcms:
            pcms[key] = scene.voice_buffer_fast(first + k)
        pcm = pcms[key]
        lib.b200mix_buffer_data(h, k, abi.FMT_I16, 1, pcm.shape[0], pcm.ctypes.data, pcm.nbytes)
    params, coeffs, pitches = bench.synth_voices(range(first, first + nv), total, lib, hrtf)
    dry = None
    for k in range(nv):
        params[k].resampler = cfg["resampler"]
        if kind != "hrtf":
            params[k].flags &= ~abi.VF_HRTF
        if nslots:
            params[k].send_slot[0] = (first + k) % nslots
    if kind != "hrtf":
        # plain first/third-order encode of the scene positions (ACN order, arbitrary norm)
        dry = np.zeros((nv, desc.dry_channels), dtype=np.float32)
        for k in range(nv):
            x, y, z = scene.voice_position(first + k)
            r = max((x * x + y * y + z * z) ** 0.5, 1e-6)
            x, y, z = x / r, y / r, z / r
            base = [1.0, y, z, x, x * y, y * z, 3 * z * z - 1, x * z, x * x - y * y,
                    y * (3 * x * x - y * y), x * y * z, y * (5 * z * z - 1), z * (5 * z * z - 3),
                    x * (5 * z * z - 1), z * (x * x - y * y), x * (x * x - 3 * y * y)]
            dry[k] = np.array(base[:desc.dry_channels], dtype=np.float32) * scene.voice_gain(total)
    send = None
    if nslots:
        send = np.zeros((nv, 1, 4), dtype=np.float32)
        send[:, 0, :] = np.array([0.5, 0.2, -0.1, 0.3], dtype=np.float32) * scene.voice_gain(total)
    assert lib.b200mix_voices_update(h, nv, params, coeffs.ctypes.data if kind == "hrtf" else None,
                                     dry.ctypes.data if dry is not None else None,
                                     send.ctypes.data if send is not None else None) == 0, \
        lib.b200mix_last_error(h)
    if args.filters:
        lp = np.zeros(5, dtype=np.float32)
        hp = np.zeros(5, dtype=np.float32)
        lib.b200mix_biquad_coeffs(0, 5000.0 / 48000.0, 0.3, 1.0, lp.ctypes.data)
        lib.b200mix_biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data)
        fl = (abi.VoiceFilter * nv)()
        for k in range(nv):
            fl[k].voice, fl[k].path, fl[k].active = k, 0, 1
            fl[k].lowpass[:] = lp.tolist()
            fl[k].highpass[:] = hp.tolist()
        assert lib.b200mix_voices_filters(h, nv, fl) == 0, lib.b200mix_last_error(h)

    stream = torch.cuda.ExternalStream(lib.b200mix_stream(h))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = C.c_void_p()
    wet_ptr, wet_cnt = C.c_void_p(), C.c_size_t()
    real_floats = desc.real_channels * 1024

    if world > 1:
        shard.connect(lib, h, rank, world, args.transport, gloo)

    def update():
        # sharded: the wet reduce-scatter and the RealOut reduce happen inside this call
        assert lib.b200mix_render_device(h, 1024, C.byref(out)) == 0, lib.b200mix_last_error(h)

    for _ in range(args.warmup):
        update()
    torch.cuda.synchronize()
    lib.b200mix_profile(h, 2)
    lib.b200mix_last_stage_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    ms, mix, stages = [], [], []
    for _ in range(args.steps):
        with torch.cuda.stream(stream):
            flush.zero_()
        if world > 1:
            torch.cuda.synchronize()
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        update()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        mix.append(lib.b200mix_last_mix_kernel_ms(h))
        st = np.zeros(8, dtype=np.float32)
        if lib.b200mix_last_stage_ms(h, st.ctypes.data, 8) == 8:
            stages.append(st)
    if args.dump_outputs and rank == 0:
        class _Block:
            __cuda_array_interface__ = {"shape": (desc.real_channels, 1024), "typestr": "<f4",
                                        "data": (out.value, False), "strides": None, "version": 2}
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, f"real_out_{args.config}.npy"),
                torch.as_tensor(_Block(), device="cuda").cpu().numpy())
    t = torch.tensor([float(np.mean(ms))], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_update = float(t.item())
    if rank == 0:
        print(json.dumps({
            "config": args.config, "kind": kind, "n_gpus": world, "voices_total": total,
            "voices_per_gpu": nv, "slots": nslots, "slots_installed_rank0": installed,
            "conv_taps": args.taps if cfg["conv"] else None,
            "transport": args.transport if world > 1 else None,
            "buffers": f"{nv} private device buffers per rank, {pool} distinct host waveforms", "direct_filters": bool(args.filters),
            "ms_per_update": ms_update, "mix_kernel_ms_rank0": float(np.mean(mix)),
            "stage_us_rank0": dict(zip(["clear", "voices", "filters+fir/deferred", "reduce", "dry_bus", "sends",
                                        "effects", "post"],
                                       [round(float(x) * 1e3, 1) for x in np.mean(stages, axis=0)]))
            if stages else None,
            "voice_samples_per_s": total * 1024 / (ms_update * 1e-3),
            "rt_voices": total * (1000.0 * 1024 / 48000) / ms_update,
            "timing": "CUDA events on the mixer stream, L2 flushed between updates, max over ranks"}))
    lib.b200mix_destroy(h)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
