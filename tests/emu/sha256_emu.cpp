// sha256_emu.cpp — TEST INFRASTRUCTURE: compiles the SHA-256 and Merkle routines of ronkathon_b200/csrc/sha256.cuh for
// the host, so the CPU test tier can check them against Python's hashlib without a GPU.  What merkle_span_kernel does
// per CTA is repeated here level by level, with the barrier between reads and writes replaced by a second buffer.
// Never linked into libronk_b200.so.
#include <cstdint>
#include <vector>

#include "../../ronkathon_b200/csrc/sha256.cuh"

using namespace ronk;

static void put_digest(const u32 h[8], uint8_t* out) {
  for (int k = 0; k < 32; k++) out[k] = (uint8_t)(h[k / 4] >> (24 - 8 * (k % 4)));
}

static void get_digest(const uint8_t* p, u32 h[8]) {
  for (int k = 0; k < 8; k++) h[k] = (u32)p[4 * k] << 24 | (u32)p[4 * k + 1] << 16 | (u32)p[4 * k + 2] << 8 | p[4 * k + 3];
}

extern "C" {

uint32_t emu_sha_k(int i) { return sha_k(i); }
uint32_t emu_sha_kw_pad64(int i) { return sha_kw_pad64(i); }

// out[32·i ..] = SHA-256 of data[off[i], off[i+1]) through sha_message, as sha256_kernel runs it.
void emu_sha256(const uint8_t* data, const uint64_t* off, uint64_t n, uint8_t* out) {
  for (uint64_t i = 0; i < n; i++) {
    u32 h[8];
    sha_message(data + off[i], off[i + 1] - off[i], h);
    put_digest(h, out + 32 * i);
  }
}

// out = digest(l ‖ r) through sha_node (a full compression, then the constant padding block).
void emu_sha_node(const uint8_t* l, const uint8_t* r, uint8_t* out) {
  u32 a[8], b[8], h[8];
  get_digest(l, a);
  get_digest(r, b);
  sha_node(a, b, h);
  put_digest(h, out);
}

// One span of cnt ≤ 512 digests reduced through nlev levels by merkle_span_node: the nodes of each level above the
// span, one level after the other, into out.  Returns the number of nodes written.
uint64_t emu_merkle_span(const uint8_t* level, uint32_t cnt, uint32_t nlev, uint8_t* out) {
  constexpr u32 S = 512;
  std::vector<u32> sm(8 * S), nx(8 * S);
  for (u32 i = 0; i < cnt; i++) {
    u32 h[8];
    get_digest(level + 32 * i, h);
    for (int k = 0; k < 8; k++) sm[k * S + i] = h[k];
  }
  uint64_t written = 0;
  for (u32 l = 1; l <= nlev; l++) {
    const u32 next = (cnt + 1) / 2;
    for (u32 t = 0; t < next; t++) {
      u32 h[8];
      merkle_span_node(sm.data(), S, t, cnt, h);
      for (int k = 0; k < 8; k++) nx[k * S + t] = h[k];
      put_digest(h, out + 32 * written++);
    }
    sm.swap(nx);
    cnt = next;
  }
  return written;
}

}  // extern "C"
