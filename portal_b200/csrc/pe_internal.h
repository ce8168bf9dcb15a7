// Internal hooks between the translation units of libportal_b200.so (not part of the C ABI).
#pragma once
#include <stddef.h>
#include <stdint.h>
struct pe_ctx;
// CUDA device ordinal of a context, -1 for a compile-only context.
int pe_internal_device(pe_ctx* ctx);
struct pe_target;
// pe_render / pe_render_rgba8 through program instance 0 or 1 (each has its own uniform block on the device): frames rendered
// through different instances on different streams may overlap.
int pe_internal_render(pe_ctx* ctx, const pe_target* target, void* out_device, void* stream, int rgba8, int instance);
// Adaptive anti-aliasing of a strip target through program instance 0 or 1 (each with its own list and halo buffers):
// pe_render_adaptive_strips without the refined count, for frames in flight on two streams.
int pe_internal_render_adaptive(pe_ctx* ctx, const pe_target* target, int threshold, int rgba8, void* out_device, void* stream,
                                int instance);
// pe_submit_host_strips_rgba8 whose device slot holds the strips of pe_render_adaptive_strips(threshold).
int pe_internal_submit_host_strips_adaptive(pe_ctx* ctx, const pe_target* target, uint8_t* host_frame, uint64_t* ticket, int threshold);
// Copy a target's compact strips (device) to their rows of a whole row-major frame (device or peer-mapped), stream-ordered:
// one pitched copy for the whole strips, one more for a ragged last strip.
int pe_internal_copy_strips(pe_ctx* ctx, const pe_target* target, void* frame_device, const void* strips_device,
                            size_t bytes_per_pixel, void* stream);
