// callback_plan.hpp — host-side planning of callback-buffer voices (AL_SOFT_callback_buffer).
//
// The reference calls a callback buffer's callback from inside the mixer's chunk loop
// (LoadResampledSamples, core/voice.cpp:726-753) and, after the mix, drops the blocks the voice
// has passed (core/voice.cpp:1155-1180).  Everything that decides those calls is integer
// arithmetic on the voice's position, fraction, step and the update size, so the library runs
// it on the host before it launches the update: the callbacks happen on the calling thread,
// the samples they deliver are shipped with the update, and the GPU reads them like a static
// span.  This header is that arithmetic, free of CUDA so that a host-only test can build it.
#pragma once
#include <cstdint>

namespace b200mix {
namespace cbplan {

constexpr uint32_t kLine = 1024;               // BufferLineSize
constexpr uint32_t kEdge = 24;                 // MaxResamplerEdge
constexpr uint32_t kPad = 48;                  // MaxResamplerPadding
constexpr uint32_t kSrcSizeMax = kLine + 256u + kPad - kEdge;   // mResampleData size - edge
constexpr uint32_t kMaxChunks = 16;            // chunks of one update at MaxPitch: 9

// CalculateBufferSize, core/voice.cpp:601-640 (the same chunking as the kernel's)
inline void buffer_size(uint32_t fracPos, uint32_t increment, uint32_t dstRemaining,
    uint32_t &dst, uint32_t &src)
{
    const uint32_t ext = increment <= 65536u;
    const uint64_t srcSize64 = ((uint64_t(dstRemaining - ext)*increment + fracPos) >> 16) + ext + kEdge;
    if(srcSize64 <= kSrcSizeMax) { dst = dstRemaining; src = uint32_t(srcSize64); return; }
    const uint64_t dstSize64 = ((uint64_t(kSrcSizeMax - kEdge)<<16) - fracPos) / increment;
    if(dstSize64 < dstRemaining) { dst = uint32_t(dstSize64) & ~3u; src = kSrcSizeMax; return; }
    dst = dstRemaining; src = kSrcSizeMax;
}

inline int32_t add_sat(int32_t a, int32_t b)
{
    const int64_t r = int64_t(a) + b;
    return r > 2147483647ll ? 2147483647 : (r < -2147483648ll ? int32_t(-2147483647 - 1) : int32_t(r));
}

// Voice::mNumCallbackBlocks, mCallbackBlockOffset and VoiceFlag::CallbackStopped
struct State { uint32_t num_blocks{0}, block_offset{0}, stopped{0}; };

// What the mixer knows of the voice at the start of an update
struct Voice {
    int32_t pos; uint32_t frac, step;
    uint32_t state;            // 0 stopped, 1 playing, 2 stopping
    bool have_buffer;          // mCurrentBuffer != nullptr
};

// The update's loads: chunk c reads `count` storage samples from cb_offset[c], those past
// num_samples[c] being the last one below it (LoadBufferCallback, core/voice.cpp:546-561);
// uint_pos[c] is the voice position the chunk starts at.  Silent chunks load nothing (count 0).
struct Loads {
    uint32_t chunks{0};
    uint32_t cb_offset[kMaxChunks]{}, num_samples[kMaxChunks]{}, uint_pos[kMaxChunks]{}, count[kMaxChunks]{};
};

// The same loads as ONE static span, which is what the GPU reads: storage sample i is span
// frame i - base, the span is `frames` frames long (0 when every load lies past the stored
// samples).  This holds because within an update cb_offset - max(position, 0) never changes
// (both advance by the same source offsets, core/voice.cpp:793-802), and a chunk's
// num_samples falls short of the update's final count only when the callback delivered all
// it was asked for, so that the chunk ends before it (tests/test_callback_plan.py checks both
// on random voices).
struct Span { int64_t base; uint32_t frames; };
inline Span span_of(const State &start, const Voice &v, uint32_t spb, const State &end)
{
    const int64_t u0 = v.pos < 0 ? 0 : v.pos;
    const int64_t base = int64_t(start.block_offset) - u0;
    const int64_t f = int64_t(end.num_blocks)*spb - base;
    if(f <= 0) return Span{0, 0u};
    return Span{base, f > 0xffffffffll ? 0xffffffffu : uint32_t(f)};
}

// Whether the voice loads anything this update (Voice::mix: a zero step returns early, a voice
// without a buffer holds its end sample).
inline bool loads_samples(const Voice &v)
{ return (v.state == 1u || v.state == 2u) && v.step >= 1u && v.have_buffer; }

// The chunk loop of LoadResampledSamples for one update of `frames` samples.  request(byte
// offset, bytes) is the callback; it returns the byte count it delivered (negative counts as 0).
// Returns false when a request would pass `storage_bytes`.
template<typename Request>
bool plan_loads(State &s, uint32_t spb, uint32_t bpb, const Voice &v, uint32_t frames,
    uint64_t storage_bytes, Request &&request, Loads &out)
{
    out.chunks = 0;
    if(!loads_samples(v)) return true;
    int32_t intPos = v.pos;
    uint32_t fracPos = v.frac, cbOffset = s.block_offset;
    const uint32_t increment = v.step;
    for(uint32_t loaded = 0;loaded < frames;)
    {
        uint32_t dstn, srcn;
        buffer_size(fracPos, increment, frames - loaded, dstn, srcn);
        bool silent = false;
        if(dstn == 0u) { dstn = frames - loaded; silent = true; }   // as the kernel (never at MaxPitch)
        uint32_t srcDelay = 0;
        if(intPos < 0)
        {
            srcDelay = uint32_t(-int64_t(intPos));
            if(srcDelay >= srcn) silent = true;
        }
        const uint32_t c = out.chunks++;
        if(c >= kMaxChunks) return false;
        if(!silent)
        {
            const uint64_t needSamples = uint64_t(cbOffset) + srcn - srcDelay;
            const uint64_t needBlocks = (needSamples + spb - 1u) / spb;
            if(!s.stopped && needBlocks > s.num_blocks)
            {
                const uint64_t byteOffset = uint64_t(s.num_blocks)*bpb;
                const uint64_t needBytes = (needBlocks - s.num_blocks)*bpb;
                if(byteOffset + needBytes > storage_bytes) return false;
                const int64_t got = request(byteOffset, uint32_t(needBytes));
                const uint64_t gotBytes = got < 0 ? 0u : uint64_t(got);
                s.stopped = needBytes != gotBytes;
                if(gotBytes <= needBytes) s.num_blocks += uint32_t(gotBytes / bpb);
            }
            out.cb_offset[c] = cbOffset;
            out.num_samples[c] = s.num_blocks*spb;
            out.uint_pos[c] = intPos < 0 ? 0u : uint32_t(intPos);
            out.count[c] = srcn - srcDelay;
        }
        loaded += dstn;
        if(loaded < frames)
        {
            fracPos += dstn*increment;
            const uint32_t srcOffset = fracPos >> 16;
            fracPos &= 0xffffu;
            if(silent) intPos = add_sat(intPos, int32_t(srcOffset));
            else if(intPos < 0)
            {
                intPos += int32_t(srcOffset);
                cbOffset += intPos < 0 ? 0u : uint32_t(intPos);
            }
            else
            {
                intPos = add_sat(intPos, int32_t(srcOffset));
                cbOffset += srcOffset;
            }
        }
    }
    return true;
}

// After the mix (core/voice.cpp:1116-1232): the voice's new position and state, and what
// happens to the stored blocks.  consumed_bytes > 0: the storage is compacted, bytes
// [consumed_bytes, consumed_bytes + kept_bytes) move to the front.  ends: the stream ran out,
// the voice stops (Stopping, no buffer), the block count and offset return to 0 and `stopped`
// stays as it is (core/voice.cpp:1174-1179).
struct After { bool ends{false}; uint64_t consumed_bytes{0}, kept_bytes{0}; };

inline After finish_update(State &s, uint32_t spb, uint32_t bpb, Voice &v, uint32_t frames)
{
    After a;
    if(v.state != 1u && v.state != 2u) return a;
    if(v.step < 1u) { if(v.state == 2u) v.state = 0u; return a; }
    if(v.state == 2u) { v.state = 0u; return a; }
    uint32_t frac = v.frac + v.step*frames;
    const uint32_t samplesDone = frac >> 16;
    v.pos = add_sat(v.pos, int32_t(samplesDone));
    v.frac = frac & 0xffffu;
    if(!v.have_buffer) { v.state = 2u; return a; }     // no buffer: Stopping (voice.cpp:1224-1232)
    if(v.pos <= 0) return a;
    const uint32_t done = samplesDone < uint32_t(v.pos) ? samplesDone : uint32_t(v.pos);
    const uint32_t endOffset = s.block_offset + done;
    const uint32_t blocksDone = endOffset / spb;
    if(blocksDone == 0u) s.block_offset = endOffset;
    else if(blocksDone < s.num_blocks)
    {
        a.consumed_bytes = uint64_t(blocksDone)*bpb;
        a.kept_bytes = uint64_t(s.num_blocks - blocksDone)*bpb;
        s.num_blocks -= blocksDone;
        s.block_offset = endOffset - blocksDone*spb;
    }
    else
    {
        a.ends = true;
        s.num_blocks = 0; s.block_offset = 0;
        v.have_buffer = false;
        v.state = 2u;
    }
    return a;
}

} // namespace cbplan
} // namespace b200mix
