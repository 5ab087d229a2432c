// ViT-encoder attention dispatch (restates segment_anything's Attention.forward + add_decomposed_rel_pos,
// oracle/sam_ref.py:Attention): the windowed blocks (14x14 windows, 196 keys incl. the zero-pad tokens, which stay in the key
// set with q=k=v=qkv.bias exactly like the reference) run attention_win2.cu, the global (64x64) blocks attention_global.cu.
#include "kernels.h"

namespace msam {

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  if (a.grid != 64) return set_error("attention: token grid %d unsupported (kernel is specialised for 64x64)", a.grid);
  if (a.window == 0) return launch_attention_global(a, stream);
  if (a.window == 14 && (a.head_dim == 64 || a.head_dim == 80)) return launch_attn_window2(a, stream);
  return set_error("attention: unsupported head_dim=%d window=%d", a.head_dim, a.window);
}

}  // namespace msam
