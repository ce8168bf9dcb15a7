// Host-callable launchers of the static helper kernels (pe_kernels.cu). Return a cudaError_t value.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace pe_host {

int launch_quantize_rgba8(const void* rgba_f32, void* rgba8, size_t n_pixels, int sms, cudaStream_t s);
int launch_deinterleave(const void* gathered, void* frame, int width, int height, int strip_rows, int n_ranks,
                        int strips_per_rank, int sms, cudaStream_t s);
int launch_signal(void* const* ptrs, int n, unsigned int value, cudaStream_t s);
int launch_average_rgba8(const void* const* frames, int n_frames, void* out, size_t n_pixels, int sms, cudaStream_t s);
// *count += number of 16-byte words in which a and b differ (bitwise); both 16-byte aligned
int launch_count_diff(const void* a, const void* b, size_t n_words16, unsigned* count, int sms, cudaStream_t s);
// Adaptive anti-aliasing: append the packed indices ((y << 16) | x) of the pixels of a whole width x height frame (RGBA8 or
// float RGBA) whose 3x3 unorm8 range exceeds `threshold` to `list`, counting them in count[0] (zeroed by the caller)
int launch_refine_list(const void* frame, bool rgba8, int width, int height, int threshold, unsigned* list, unsigned* count,
                       cudaStream_t s);

}  // namespace pe_host
