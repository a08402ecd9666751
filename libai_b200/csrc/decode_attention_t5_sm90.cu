// The T5 instances of the split-KV decode attention kernel: the decoder self-attention with the relative-position bias
// (Score::kRelBias) and the cross-attention over the encoder's keys (Score::kWindow), kept in their own translation unit
// so that the objects of decode_attention_sm90.cu and decode_attention_alibi_sm90.cu hold exactly the kernels they held
// before them.
#include "decode_attention_sm90.cuh"

namespace lb {
namespace dec {

cudaError_t launch_decode_attn_t5(const Params& p, Score S, int D, int B, int nsplit, cudaStream_t s) {
  if (S == Score::kRelBias)
    return D == 64 ? launch_decode_attn<64, Score::kRelBias>(p, B, nsplit, s)
                   : launch_decode_attn<128, Score::kRelBias>(p, B, nsplit, s);
  return D == 64 ? launch_decode_attn<64, Score::kWindow>(p, B, nsplit, s)
                 : launch_decode_attn<128, Score::kWindow>(p, B, nsplit, s);
}

}  // namespace dec
}  // namespace lb
