// The library's callback-buffer planner (openal-soft_b200/csrc/callback_plan.hpp) built for the
// host, for tests/test_callback_plan.py: one update of one voice, with the callback answered by
// the caller.
#include <cstdint>

#include "../../openal-soft_b200/csrc/callback_plan.hpp"

using namespace b200mix;

extern "C" {

typedef int64_t (*cbplan_request_fn)(uint64_t offset, uint32_t bytes);

struct cbplan_update {
    // in/out: the buffer state and the voice
    uint32_t num_blocks, block_offset, stopped;
    int32_t pos; uint32_t frac, step, state, have_buffer;
    // out
    uint32_t chunks;
    uint32_t cb_offset[cbplan::kMaxChunks], num_samples[cbplan::kMaxChunks];
    uint32_t uint_pos[cbplan::kMaxChunks], count[cbplan::kMaxChunks];
    int64_t span_base; uint32_t span_frames;
    uint32_t ends; uint64_t consumed_bytes, kept_bytes;
};

__attribute__((visibility("default")))
int cbplan_run(cbplan_update *u, uint32_t spb, uint32_t bpb, uint32_t frames, uint64_t storage_bytes,
    cbplan_request_fn request)
{
    cbplan::State st{u->num_blocks, u->block_offset, u->stopped};
    cbplan::Voice v{u->pos, u->frac, u->step, u->state, u->have_buffer != 0};
    const cbplan::State start = st;
    cbplan::Loads loads;
    if(!cbplan::plan_loads(st, spb, bpb, v, frames, storage_bytes, request, loads)) return -1;
    const cbplan::Span span = cbplan::span_of(start, v, spb, st);
    const cbplan::After after = cbplan::finish_update(st, spb, bpb, v, frames);
    u->chunks = loads.chunks;
    for(uint32_t c = 0;c < loads.chunks;++c)
    {
        u->cb_offset[c] = loads.cb_offset[c]; u->num_samples[c] = loads.num_samples[c];
        u->uint_pos[c] = loads.uint_pos[c]; u->count[c] = loads.count[c];
    }
    u->span_base = span.base; u->span_frames = span.frames;
    u->ends = after.ends; u->consumed_bytes = after.consumed_bytes; u->kept_bytes = after.kept_bytes;
    u->num_blocks = st.num_blocks; u->block_offset = st.block_offset; u->stopped = st.stopped;
    u->pos = v.pos; u->frac = v.frac; u->state = v.state; u->have_buffer = v.have_buffer;
    return 0;
}

}
