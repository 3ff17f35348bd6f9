// tc_ptx.cuh -- inline-PTX wrappers: mbarrier, TMA (tiled loads and stores, bulk copies), wgmma shared-memory descriptors
// Part of the tensor-core engine's single translation unit: included by kernels_tc.cu inside namespace w2x::tc, in this order:
//   tc_ptx.cuh, tc_wgmma.cuh, tc_config.cuh, tc_kernel.cuh, tc_edge_kernels.cuh
// (pure code organisation: the generated SASS is the same as with one file).

// ================================================================================================
// PTX wrappers
// ================================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
// Producer-side helpers are called by a whole converged warp; ONE elected lane executes the instruction (elect.sync inside
// the asm block).  For the TMA instructions this is what lets ptxas keep their operands in uniform registers.
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Spin on try_wait; a protocol bug must not hang the GPU, so give up (trap -> launch error) after ~4 s.  The whole loop is
// one asm block: a __trap() in the C++ control flow makes ptxas serialise the wgmmas that are in flight across the wait.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        ".reg .u64 t0, t1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "mov.u64 t0, %%clock64;\n"
        "WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "mov.u64 t1, %%clock64;\n\t"
        "sub.u64 t1, t1, t0;\n\t"
        "setp.lt.u64 p, t1, 8000000000;\n\t"
        "@p bra WAIT;\n\t"
        "trap;\n"
        "DONE:\n\t"
        "}" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of `count` threads (the two consumer warpgroups synchronise separately: ids 1 and 2)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// TMA: 4-D tiled load global -> shared, completion on an mbarrier
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t@q cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n\t}"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// bulk (1-D) copy global -> shared, completion on an mbarrier
__device__ __forceinline__ void bulk_load(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t@q cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}" ::"r"(dst),
                 "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
                 : "memory");
}
// TMA store of one 4-D box shared -> global (bulk async-group completion); whole warp calls, one elected lane issues
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t@q cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n\t}"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() {
    asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t@q cp.async.bulk.commit_group;\n\t}" ::: "memory");
}
// Every lane waits for ITS OWN bulk groups (lanes that issued none return at once), so whichever lane the elect.sync of
// tma_store_4d / bulk_commit picked is covered; callers follow with __syncwarp().
// ... have finished READING shared memory (the staging tile may be rewritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... have completed (before the CTA exits)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// Per-thread register limit of the executing warpgroup (all four warps execute it, converged): .dec hands registers back
// to the CTA's pool, .inc waits until the pool holds enough and takes them.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}

// ================================================================================================
// Descriptors
// ================================================================================================
// wgmma shared-memory matrix descriptor (K-major, swizzled), PTX ISA "Matrix Descriptor Format": start address >>4 in
// [0,14), leading byte offset >>4 in [16,30) (unused for swizzled K-major; written as 1), stride byte offset >>4 in [32,46),
// base offset in [49,52) (0: every swizzle pattern here starts 1024-byte aligned), layout type in [62,64)
// (1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B).
// Canonical K-major layout, 16-byte units: ((8, n), 2) : ((ROWB/16, SBO), 1) -- eight rows ROWB bytes apart form a group,
// groups are SBO bytes apart, the swizzle XOR is a function of the shared-memory ADDRESS bits, which is what lets a
// descriptor start at any row inside a TMA-written box (the 3x3 taps are start-address offsets).
enum : uint32_t { SW128 = 1u, SW64 = 2u, SW32 = 3u };

// Everything of a descriptor except the start address: the high word.
__host__ __device__ constexpr uint32_t desc_hi(uint32_t sbo_bytes, uint32_t layout_type) {
    return ((sbo_bytes >> 4) & 0x3FFFu) | (layout_type << 30);
}
__device__ __forceinline__ uint64_t make_desc(uint32_t hi32, uint32_t saddr) {
    return ((uint64_t)hi32 << 32) | (uint64_t)(((saddr >> 4) & 0x3FFFu) | (1u << 16));
}
