// inflate_slow.cu — generic serial Deflate decoder, one thread per unit, for the (malformed) streams the fast path
// cannot take: Huffman code sets whose Kraft sum exceeds 1.  The reference accepts those: Code.huffmanCodes never
// validates (Sources/Common/CodingTree/Code.swift:15-39), DecodingTree.init overwrites heap slots
// (DecodingTree.swift:22-32) and findNextSymbol returns at the first leaf on the path (:36-50) — so "shortest prefix
// wins, and among equal paths the code assigned last wins".  That rule is emulated here directly on the sorted code
// list (no 2^16-slot heap per tree).  Only units the Huffman stage (K1L / K1w) flagged SWC_INTERNAL_NEEDS_SLOW are touched.
#include "common.cuh"
#include "inflate_serial.cuh"

namespace swc {
namespace inflate {

__global__ void __launch_bounds__(64) inflate_slow_kernel(BatchArgs a) {
    const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (unit >= a.n) return;
    if (a.status[unit] != SWC_INTERNAL_NEEDS_SLOW) return;
    u64 op = 0, used = 0;
    a.status[unit] = inflate_serial(a.in_base + a.in_off[unit], a.in_len[unit] * 8, a.start_bits ? a.start_bits[unit] : 0,
                                    a.out_base + a.out_off[unit], a.out_cap[unit], &op, &used);
    a.out_len[unit] = op;
    a.consumed[unit] = used;
    a.rec_count[unit] = REC_DIRECT;      // the output is written: K2 leaves the unit alone
}

void launch_slow(const BatchArgs &a, cudaStream_t stream) {
    inflate_slow_kernel<<<(unsigned)((a.n + 63) / 64), 64, 0, stream>>>(a);
    count_launch();
}

}  // namespace inflate
}  // namespace swc
