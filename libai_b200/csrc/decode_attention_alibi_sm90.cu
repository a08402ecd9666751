// The ALiBi instances of the split-KV decode attention kernel (BLOOM), kept in their own translation unit so that the
// object of decode_attention_sm90.cu holds exactly the kernels it held before them.
#include "decode_attention_sm90.cuh"

namespace lb {
namespace dec {

cudaError_t launch_decode_attn_alibi(const Params& p, int D, int B, int nsplit, cudaStream_t s) {
  return D == 64 ? launch_decode_attn<64, Score::kAlibi>(p, B, nsplit, s)
                 : launch_decode_attn<128, Score::kAlibi>(p, B, nsplit, s);
}

}  // namespace dec
}  // namespace lb
