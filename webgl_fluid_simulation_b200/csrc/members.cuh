// members.cuh — the member-subset data calls of batch handles (fluid_read_members / fluid_write_members with a
// device buffer, fluid_reset_members).  Every launch takes the listed members as grid z: layer z of blocks works
// on member list[z], which the host checked and uploaded.  A member of a batch field is one contiguous block of
// the field's dense (B, H, W[, C]) array; batch rows are at least 128 floats wide, so every member block starts
// 16-byte aligned and holds a whole number of float4.  Offsets are 64-bit: a (B, 1024, 1024, 4) dye passes 2^32
// bytes once B > 256.
#pragma once
#include <cuda_runtime.h>

namespace fk {

// Copies member list[z]'s block of `per` V's between a field and slot z of a caller's dense (n, per) buffer.
// TO_BUF: field -> buffer (the gather of a read), else buffer -> field (the scatter of a write).  V: float4 when
// the caller's buffer is 16-byte aligned, float when it is only 4-byte aligned; any field width either way.
template <class V, bool TO_BUF>
__global__ void __launch_bounds__(256) member_copy_kernel(const V* __restrict__ src, V* __restrict__ dst,
                                                          const int* __restrict__ list, size_t per) {
    const size_t m = (size_t)__ldg(list + blockIdx.z), z = blockIdx.z;
    src += (TO_BUF ? m : z) * per;
    dst += (TO_BUF ? z : m) * per;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < per; k += stride) dst[k] = src[k];
}

// Every slot of a batch handle's arena, as float4 arrays of `per` float4 per member: both dye slots first, whose
// cells reset to alpha 1, then both velocity and pressure slots, divergence and curl, which reset to zero.
struct MemberSlots {
    float4* p[8];
    size_t per[8];
};

// member list[z] back to the state fluid_create_batch leaves (make_arena: zero, dye alpha 1), every slot of it
// in one launch
__global__ void __launch_bounds__(256) member_reset_kernel(MemberSlots s, const int* __restrict__ list) {
    const size_t m = (size_t)__ldg(list + blockIdx.z);
    const size_t k0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const float4 v = make_float4(0.f, 0.f, 0.f, r < 2 ? 1.f : 0.f);
        float4* const p = s.p[r] + m * s.per[r];
        for (size_t k = k0; k < s.per[r]; k += stride) p[k] = v;
    }
}

}  // namespace fk
