// Key-set geometry of the temporal focal window attention, shared by the forward (focal_attn.cu) and its backward
// (focal_attn_grad.cu): which expanded-window positions the reference lists as keys, and how often.
#pragma once
#include <cstdint>

namespace e2f {
namespace attn {

constexpr int MAX_RING = 256;                  // expanded-window positions (153 for the 5x9 window)

// how many times the reference lists expanded-window position (er, ec) as a key (tfocal_transformer.py:166-179,235-280)
__host__ __device__ inline int key_multiplicity(int er, int ec, int wh, int ww, int eh, int ew) {
  int m = 0;
  if (er >= eh && er < eh + wh && ec >= ew && ec < ew + ww) m += 1;                      // own window
  {  // tl: window pos (r,c) holds token (r+eh, c+ew) -> expanded (r+2eh, c+2ew); kept if r>=wh-eh or c>=ww-ew
    const int r = er - 2 * eh, c = ec - 2 * ew;
    if (r >= 0 && r < wh && c >= 0 && c < ww && (r >= wh - eh || c >= ww - ew)) m += 1;
  }
  {  // tr: expanded (r+2eh, c); kept if r>=wh-eh or c<ew
    const int r = er - 2 * eh, c = ec;
    if (r >= 0 && r < wh && c >= 0 && c < ww && (r >= wh - eh || c < ew)) m += 1;
  }
  {  // bl: expanded (r, c+2ew); kept if r<eh or c>=ww-ew
    const int r = er, c = ec - 2 * ew;
    if (r >= 0 && r < wh && c >= 0 && c < ww && (r < eh || c >= ww - ew)) m += 1;
  }
  {  // br: expanded (r, c); kept if r<eh or c<ew
    const int r = er, c = ec;
    if (r >= 0 && r < wh && c >= 0 && c < ww && (r < eh || c < ew)) m += 1;
  }
  return m;
}

// Orders the expanded-window positions the reference lists: the n1 listed once first, then the n2 listed more than once
// (positions never listed are dropped).  pos / mult receive n1 + n2 entries; EH * EW <= MAX_RING.
inline void order_ring(int wh, int ww, int eh, int ew, uint8_t* pos, uint8_t* mult, int& n1, int& n2) {
  const int EH = wh + 2 * eh, EW = ww + 2 * ew;
  n1 = n2 = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int e = 0; e < EH * EW; ++e) {
      const int m = key_multiplicity(e / EW, e % EW, wh, ww, eh, ew);
      if ((pass == 0 && m == 1) || (pass == 1 && m > 1)) {
        const int slot = n1 + n2;
        pos[slot] = static_cast<uint8_t>(e);
        mult[slot] = static_cast<uint8_t>(m);
        (pass == 0 ? n1 : n2)++;
      }
    }
}

}  // namespace attn
}  // namespace e2f
