"""The library's callback-buffer planner (openal-soft_b200/csrc/callback_plan.hpp, built for the host as
libcbplan_host.so) against a separate Python restatement of the reference's callback loading
(LoadResampledSamples' IsCallback branch, core/voice.cpp:726-753 and :793-802; the post-mix block
consumption, :1155-1180).  Seeded random positions, fractions, steps up to MaxPitch, update sizes,
block sizes and short callback returns.  Same request sequence (byte offset and count), same
state, position and end decision.  The single span the GPU reads matches every chunk's loads."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_CHUNKS = 16
EDGE, SRC_MAX = 24, 1024 + 256 + 48 - 24

REQUEST_FN = C.CFUNCTYPE(C.c_int64, C.c_uint64, C.c_uint32)


class Update(C.Structure):
    _fields_ = [("num_blocks", C.c_uint32), ("block_offset", C.c_uint32), ("stopped", C.c_uint32),
                ("pos", C.c_int32), ("frac", C.c_uint32), ("step", C.c_uint32), ("state", C.c_uint32),
                ("have_buffer", C.c_uint32), ("chunks", C.c_uint32),
                ("cb_offset", C.c_uint32 * MAX_CHUNKS), ("num_samples", C.c_uint32 * MAX_CHUNKS),
                ("uint_pos", C.c_uint32 * MAX_CHUNKS), ("count", C.c_uint32 * MAX_CHUNKS),
                ("span_base", C.c_int64), ("span_frames", C.c_uint32),
                ("ends", C.c_uint32), ("consumed_bytes", C.c_uint64), ("kept_bytes", C.c_uint64)]


def _lib():
    lib = C.CDLL(os.path.join(ROOT, "openal-soft_b200", "libcbplan_host.so"))
    lib.cbplan_run.argtypes = [C.POINTER(Update), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, REQUEST_FN]
    lib.cbplan_run.restype = C.c_int
    return lib


def _sat(v):
    return max(-2**31, min(2**31 - 1, v))


def reference_update(st, voice, spb, bpb, frames, answer):
    """One Voice::mix of a callback voice, restated from the reference.  st: dict num_blocks,
    block_offset, stopped; voice: dict pos, frac, step, state, have; answer(offset, bytes) -> returned.
    Returns (requests, loads) where loads = [(cb_offset, count, num_samples)] per loading chunk."""
    requests, loads = [], []
    if voice["state"] not in (1, 2) or voice["step"] < 1:
        if voice["state"] == 2 and voice["step"] < 1:
            voice["state"] = 0
        return requests, loads
    inc = voice["step"]
    if voice["have"]:
        int_pos, frac, cb_off = voice["pos"], voice["frac"], st["block_offset"]
        done = 0
        while done < frames:
            remaining = frames - done
            ext = 1 if inc <= 65536 else 0
            src = (((remaining - ext) * inc + frac) >> 16) + ext + EDGE
            dst = remaining
            if src > SRC_MAX:
                d64 = (((SRC_MAX - EDGE) << 16) - frac) // inc
                dst, src = (d64 & ~3, SRC_MAX) if d64 < remaining else (remaining, SRC_MAX)
            delay = -int_pos if int_pos < 0 else 0
            if delay >= src:
                done += dst
                if done < frames:
                    frac += dst * inc
                    int_pos = _sat(int_pos + (frac >> 16))
                    frac &= 0xffff
                continue
            need_blocks = (cb_off + src - delay + spb - 1) // spb
            if not st["stopped"] and need_blocks > st["num_blocks"]:
                off = st["num_blocks"] * bpb
                need = (need_blocks - st["num_blocks"]) * bpb
                got = max(0, answer(off, need))
                requests.append((off, need, got))
                st["stopped"] = int(need != got)
                if got <= need:
                    st["num_blocks"] += got // bpb
            loads.append((cb_off, src - delay, st["num_blocks"] * spb, max(int_pos, 0)))
            done += dst
            if done < frames:
                frac += dst * inc
                off = frac >> 16
                frac &= 0xffff
                if int_pos < 0:
                    int_pos += off
                    cb_off += max(int_pos, 0)
                else:
                    int_pos = _sat(int_pos + off)
                    cb_off += off
    if voice["state"] == 2:
        voice["state"] = 0
        return requests, loads
    frac = voice["frac"] + inc * frames
    samples_done = frac >> 16
    voice["pos"] = _sat(voice["pos"] + samples_done)
    voice["frac"] = frac & 0xffff
    if voice["have"] and voice["pos"] > 0:
        end_off = st["block_offset"] + min(samples_done, voice["pos"])
        blocks_done = end_off // spb
        if blocks_done == 0:
            st["block_offset"] = end_off
        elif blocks_done < st["num_blocks"]:
            st["num_blocks"] -= blocks_done
            st["block_offset"] = end_off - blocks_done * spb
        else:
            st["num_blocks"] = st["block_offset"] = 0
            voice["have"] = False
            voice["state"] = 2
    return requests, loads


# (samples per block, bytes per block): PCM mono i16 / stereo f32, IMA4 mono spb 65, MSADPCM stereo spb 64
FORMATS = [(1, 2), (1, 8), (65, 36), (64, 70)]


@pytest.mark.parametrize("seed", range(6))
def test_planner_matches_reference_restatement(seed):
    lib = _lib()
    rng = np.random.default_rng(9100 + seed)
    cases = 0
    for _ in range(150):
        spb, bpb = FORMATS[int(rng.integers(len(FORMATS)))]
        step = int(rng.choice([int(rng.integers(1, 10 << 16)), 65536, 45875, 111411, 216268, 10 << 16]))
        st = {"num_blocks": 0, "block_offset": 0, "stopped": 0}
        voice = {"pos": int(rng.choice([0, 0, int(rng.integers(-3000, 0))])),
                 "frac": int(rng.integers(0, 65536)) if rng.random() < 0.7 else 0,
                 "step": step, "state": 1, "have": True}
        stream_bytes = int(rng.integers(0, 400000)) if rng.random() < 0.5 else 1 << 40
        # PrepareCallback's size (al/buffer.cpp:468-473): MixerLineSize (1024 + 256) * MaxPitch + 24
        storage = (((1024 + 256) * 10 + 24 + spb - 1) // spb) * bpb
        fed = [0, 0]                                   # bytes fed so far: reference, planner

        def make_answer(k):
            def answer(offset, need):
                got = min(need, max(0, stream_bytes - fed[k]))
                fed[k] += got
                return got
            return answer

        ref_answer, lib_calls = make_answer(0), []
        lib_answer = make_answer(1)

        @REQUEST_FN
        def request(offset, need):
            got = lib_answer(int(offset), int(need))
            lib_calls.append((int(offset), int(need), got))
            return got

        u = Update(0, 0, 0, voice["pos"], voice["frac"], step, 1, 1)
        for upd in range(12):
            if voice["state"] == 0:
                break
            frames = int(rng.choice([1, 7, 333, 1024, int(rng.integers(1, 1025))]))
            if rng.random() < 0.1 and voice["state"] == 1:
                voice["state"] = u.state = 2               # stopping (pause / stop): one fade-out update
            lib_calls.clear()
            had, was_playing = voice["have"], voice["state"] == 1
            requests, loads = reference_update(st, voice, spb, bpb, frames, ref_answer)
            assert lib.cbplan_run(C.byref(u), spb, bpb, frames, storage, request) == 0
            what = f"seed {seed} spb {spb} step {step} update {upd} frames {frames}"
            assert lib_calls == requests, what
            assert (u.num_blocks, u.block_offset, u.stopped) == (st["num_blocks"], st["block_offset"],
                                                                st["stopped"]), what
            assert (u.pos, u.frac, u.state, bool(u.have_buffer)) == (voice["pos"], voice["frac"], voice["state"],
                                                                    voice["have"]), what
            assert bool(u.ends) == (had and not voice["have"]), what
            # the one span the GPU reads reproduces every chunk's LoadBufferCallback
            final = loads[-1][2] if loads else 0
            chunk_loads = [(u.cb_offset[c], u.count[c], u.num_samples[c], u.uint_pos[c])
                           for c in range(u.chunks) if u.count[c]]
            assert chunk_loads == loads, what
            for cb_off, count, num, upos in loads:
                assert cb_off == upos + u.span_base, what
                assert cb_off + count <= num or num == final, what
            if loads:
                assert u.span_frames == max(0, final - u.span_base), what
                # the GPU's static end check on the span is the reference's block rule
                if was_playing:
                    assert bool(u.ends) == (u.pos > 0 and u.pos >= u.span_frames), what
            cases += 1
    assert cases > 300
