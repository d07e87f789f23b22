// Device helpers shared by the int4 kernels (qmatvec.cu, decode_mega.cu, qgemm_wgmma.cu, qgemm_wgmma_t.cu): asynchronous staging,
// reference-exact int4 -> fp16 dequantisation, and the swapped-operand m16n8k16 tensor-core dot.
#pragma once
#include "common.cuh"

namespace gptq {
namespace int4 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
    return r;
}
// ---- mbarrier + bulk asynchronous copy (TMA unit, no tensor map: contiguous bytes global -> shared) -----------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// for waits that are expected to be long (a producer facing a full ring): sleep between probes instead of spinning
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(200);
}
// `bytes` (multiple of 16) contiguous bytes global -> shared; completion is signalled on `bar` (complete_tx); `policy`: L2 cache policy
// (createpolicy) of the lines read
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(bar), "l"(policy)
                 : "memory");
}

__device__ __forceinline__ float ld_cg(const float* p) {
    float r;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 ld_cg4(const float* p) {
    float4 r;
    asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ __half ld_cg_h(const __half* p) {
    unsigned short r;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return __ushort_as_half(r);
}
__device__ __forceinline__ uint4 ld_cg_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

__device__ __forceinline__ uint32_t h2_as_u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 u32_as_h2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }

__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Per-group dequant constants of one lane's 4 columns.
struct GroupConst {
    __half2 za01, za23;  // 1024 + z   for columns (0,1) and (2,3);  z = stored zero + 1
    __half2 zb01, zb23;  // -(64 + z)
    __half2 s01, s23;    // fp16 scales
};

// raw scale / zero words of one group for the lane's 4 columns
struct GroupRaw {
    uint2 s;     // 4 fp16 scales
    uint32_t z;  // qzeros word holding the 4 nibbles
};

__device__ __forceinline__ GroupRaw load_group_raw(const __half* __restrict__ sc, const uint32_t* __restrict__ qz) {
    GroupRaw r;
    r.s = __ldg(reinterpret_cast<const uint2*>(sc));
    r.z = __ldg(qz);
    return r;
}

__device__ __forceinline__ void build_group_const(GroupConst& c, const GroupRaw& r, int zshift) {
    const uint32_t zw = (r.z >> zshift) & 0xffffu;  // nibbles of columns col..col+3
    const __half2 one = __float2half2_rn(1.0f), c960 = __float2half2_rn(960.0f);
    uint32_t z01, z23;  // (1024+z0', 1024+z1'), (1024+z2', 1024+z3')
    asm("lop3.b32 %0, %1, %2, 0x000f000f, 0xa8;" : "=r"(z01) : "r"(zw), "r"(zw << 12));  // (a | b) & c
    asm("lop3.b32 %0, %1, %2, 0x000f000f, 0xa8;" : "=r"(z23) : "r"(zw >> 8), "r"(zw << 4));
    z01 |= 0x64006400u;
    z23 |= 0x64006400u;
    c.za01 = __hadd2(u32_as_h2(z01), one);  // +1: zeros are stored minus one, the +1 is unmasked (quant_linear.py:120-121)
    c.za23 = __hadd2(u32_as_h2(z23), one);
    c.zb01 = __hsub2(c960, c.za01);  // 960 - (1024 + z) = -(64 + z)
    c.zb23 = __hsub2(c960, c.za23);
    c.s01 = u32_as_h2(r.s.x);
    c.s23 = u32_as_h2(r.s.y);
}

template <int HI>
__device__ __forceinline__ __half2 bcast(__half2 v) {  // folds into the .H0_H0 / .H1_H1 operand modifiers
    return HI ? __half2half2(__high2half(v)) : __half2half2(__low2half(v));
}

// (q & mask) | 0x64006400 in ONE LOP3 (written as and+or the compiler emits two: LOP3 encodes a single immediate)
template <uint32_t MASK>
__device__ __forceinline__ __half2 nibbles_to_h2(uint32_t q) {
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, 0x64006400, 0xea;" : "=r"(r) : "r"(q), "n"(MASK));
    return u32_as_h2(r);
}

template <int HI>
__device__ __forceinline__ void dequant8(uint32_t q, __half2 za_pair, __half2 zb_pair, __half2 s_pair, uint32_t (&w)[4]) {
    const __half2 za = bcast<HI>(za_pair), zb = bcast<HI>(zb_pair), s = bcast<HI>(s_pair);
    const __half2 sixteenth = __float2half2_rn(0.0625f);
    const uint32_t q8 = q >> 8;
    const __half2 l0 = nibbles_to_h2<0x000f000fu>(q);   // 1024 + n
    const __half2 h0 = nibbles_to_h2<0x00f000f0u>(q);   // 1024 + 16 n
    const __half2 l1 = nibbles_to_h2<0x000f000fu>(q8);
    const __half2 h1 = nibbles_to_h2<0x00f000f0u>(q8);
    w[0] = h2_as_u32(__hmul2(__hsub2(l0, za), s));
    w[1] = h2_as_u32(__hmul2(__hfma2(h0, sixteenth, zb), s));
    w[2] = h2_as_u32(__hmul2(__hsub2(l1, za), s));
    w[3] = h2_as_u32(__hmul2(__hfma2(h1, sixteenth, zb), s));
}

// dequant8's zero constants of one column from its qzeros word: za = 1024 + z, zb = -(64 + z)
__device__ __forceinline__ void zero_consts(uint32_t zw, int zshift, __half2& za, __half2& zb) {
    const float z = (float)(((zw >> zshift) & 0xfu) + 1u);  // stored minus one, +1 unmasked (quant_linear.py:120-121)
    za = __float2half2_rn(1024.f + z);
    zb = __float2half2_rn(-(64.f + z));
}

// one packed word (8 consecutive k of one column) dequantised into a 16-byte chunk of halves in natural k order (a wgmma B-tile chunk)
__device__ __forceinline__ uint4 dequant_chunk(uint32_t q, __half2 za, __half2 zb, __half2 s) {
    uint32_t v[4];  // (k0,k4) (k1,k5) (k2,k6) (k3,k7)
    dequant8<0>(q, za, zb, s, v);
    uint4 o;
    o.x = __byte_perm(v[0], v[1], 0x5410);  // (k0,k1)
    o.y = __byte_perm(v[2], v[3], 0x5410);  // (k2,k3)
    o.z = __byte_perm(v[0], v[1], 0x7632);  // (k4,k5)
    o.w = __byte_perm(v[2], v[3], 0x7632);  // (k6,k7)
    return o;
}

}  // namespace int4
}  // namespace gptq
