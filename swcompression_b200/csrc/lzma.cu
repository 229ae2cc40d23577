// lzma.cu — batched LZMA / LZMA2 decode for sm_90a.  Replaces LZMADecoder.decode (reference
// Sources/LZMA/LZMADecoder.swift:107-298), LZMARangeDecoder (LZMARangeDecoder.swift:20-80), the bit-tree / length
// decoders (LZMABitTreeDecoder.swift, LZMALenDecoder.swift) and LZMA2Decoder (Sources/LZMA2/LZMA2Decoder.swift:17-99).
//
// ONE WARP PER UNIT.  The adaptive range coder is a strictly serial chain, so the 32 lanes execute it in lock-step
// (identical state in every lane, uniform control flow); what the warp buys is (a) the probability model — isMatch/
// isRep/posSlot/align/len tables and up to 16 literal coders, 28 KB of 11-bit counters — living in shared memory as
// u16, (b) the compressed stream arriving 128 B at a time through one coalesced, double-buffered load and (c) match
// copies done by all lanes.  The output buffer doubles as the dictionary (the reference never wraps it either).
#include "common.cuh"
#include "lzma.cuh"
#include "lzma_dec.cuh"
#include "host_util.h"

namespace swc {
namespace lzma {

__global__ void __launch_bounds__(WARPS * 32) lzma_kernel(Args a) {
    extern __shared__ u16 smem16[];
    const u32 warp = threadIdx.x >> 5;
    const u64 unit = (u64)blockIdx.x * WARPS + warp;
    if (unit >= a.n) return;
    Dec d;
    d.start(smem16 + warp * SMEM_U16, a.out_base + a.out_off[unit], a.out_cap[unit]);
    u16 *lit_global = a.lit_scratch ? a.lit_scratch + unit * ((size_t)1 << 12) * 0x300 : nullptr;
    const u8 *in = a.in_base + a.in_off[unit];
    const u64 in_len = a.in_len[unit];
    d.in_init(in, in_len);
    const u64 addr0 = d.addr;
    int st = SWC_OK;

    if (a.mode == MODE_RAW) {
        const u32 pr = a.props[unit];
        d.lc = pr & 0xFF; d.lp = (pr >> 8) & 0xFF; d.pb = (pr >> 16) & 0xFF;
        d.dict_size = a.dict_size[unit];
        d.usize = a.usize[unit] < 0 ? -1 : a.usize[unit];
        // no properties byte holds these; the reference decodes some such streams (Swift's >> by a negative count shifts
        // left) and traps on others, the engine takes none of them (DESIGN §6)
        if (d.lc > 8 || d.lp > 4 || d.pb > 4) st = SWC_ERR_UNSUPPORTED;
        else { d.reset_state(lit_global); st = d.decode(); }
    } else {
        st = lzma2_decode(d, a.dict_bytes[unit], lit_global);
    }
    if (lane_id() == 0) {
        a.out_len[unit] = (u64)d.dict_end;
        a.consumed[unit] = d.addr - addr0;
        a.status[unit] = st;
    }
}

static int configure() {
    return configure_once(CFG_LZMA, [](DeviceCtx &) {
        SWC_CUDA_TRY(cudaFuncSetAttribute(lzma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        return (int)SWC_OK;
    });
}

int occupancy_blocks(int *blocks) {
    if (int st = configure()) return st;
    SWC_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, lzma_kernel, WARPS * 32, SMEM_BYTES));
    return SWC_OK;
}

int launch(const Args &a, cudaStream_t stream) {
    if (a.n == 0) return SWC_OK;
    if (int st = configure()) return st;
    lzma_kernel<<<(unsigned)((a.n + WARPS - 1) / WARPS), WARPS * 32, SMEM_BYTES, stream>>>(a);
    count_launch();
    SWC_CUDA_TRY(cudaGetLastError());
    return SWC_OK;
}

}  // namespace lzma
}  // namespace swc
