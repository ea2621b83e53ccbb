// sha256.cuh — the reference's SHA-256 (src/hashes/sha.rs:88-201, standard FIPS 180 SHA-256) on one message per thread,
// and the node step of its Merkle tree (src/tree/merkle.rs:31-60).  Host-compilable (RONK_DEV), so tests/emu can run
// the very routines the kernels of sha256.cu run.
//
// - Compression keeps the eight state words and a 16-word schedule window in registers: the 64 rounds are unrolled,
//   so every K[i] is an immediate and the window index i mod 16 a register name.  Rotates are funnel shifts; ch and maj
//   are written as plain and/xor/not, which the compiler folds into one LOP3 each.
// - A node hashes L ‖ R, 64 bytes, so its second block is always the padding block (0x80, zeros, bit length 512).  Its
//   schedule is a constant: sha_kw_pad64 holds K[i] + W[i] for it, and that compression runs no schedule.
// - A message is read from its own bytes only: aligned 32-bit words inside [start, end), assembled into the big-endian
//   words at any start alignment with one byte permute each; the aligned word that holds the first or the last byte
//   of the message (when that word is partial) is gathered byte by byte.  Padding is formed in registers.
#pragma once
#include "field.cuh"

namespace ronk {

// K[i] (FIPS 180-4 §4.2.2)
#define RONK_SHA256_K(X)                                                                                              \
  X(0, 0x428a2f98u) X(1, 0x71374491u) X(2, 0xb5c0fbcfu) X(3, 0xe9b5dba5u)                                             \
  X(4, 0x3956c25bu) X(5, 0x59f111f1u) X(6, 0x923f82a4u) X(7, 0xab1c5ed5u)                                             \
  X(8, 0xd807aa98u) X(9, 0x12835b01u) X(10, 0x243185beu) X(11, 0x550c7dc3u)                                           \
  X(12, 0x72be5d74u) X(13, 0x80deb1feu) X(14, 0x9bdc06a7u) X(15, 0xc19bf174u)                                         \
  X(16, 0xe49b69c1u) X(17, 0xefbe4786u) X(18, 0x0fc19dc6u) X(19, 0x240ca1ccu)                                         \
  X(20, 0x2de92c6fu) X(21, 0x4a7484aau) X(22, 0x5cb0a9dcu) X(23, 0x76f988dau)                                         \
  X(24, 0x983e5152u) X(25, 0xa831c66du) X(26, 0xb00327c8u) X(27, 0xbf597fc7u)                                         \
  X(28, 0xc6e00bf3u) X(29, 0xd5a79147u) X(30, 0x06ca6351u) X(31, 0x14292967u)                                         \
  X(32, 0x27b70a85u) X(33, 0x2e1b2138u) X(34, 0x4d2c6dfcu) X(35, 0x53380d13u)                                         \
  X(36, 0x650a7354u) X(37, 0x766a0abbu) X(38, 0x81c2c92eu) X(39, 0x92722c85u)                                         \
  X(40, 0xa2bfe8a1u) X(41, 0xa81a664bu) X(42, 0xc24b8b70u) X(43, 0xc76c51a3u)                                         \
  X(44, 0xd192e819u) X(45, 0xd6990624u) X(46, 0xf40e3585u) X(47, 0x106aa070u)                                         \
  X(48, 0x19a4c116u) X(49, 0x1e376c08u) X(50, 0x2748774cu) X(51, 0x34b0bcb5u)                                         \
  X(52, 0x391c0cb3u) X(53, 0x4ed8aa4au) X(54, 0x5b9cca4fu) X(55, 0x682e6ff3u)                                         \
  X(56, 0x748f82eeu) X(57, 0x78a5636fu) X(58, 0x84c87814u) X(59, 0x8cc70208u)                                         \
  X(60, 0x90befffau) X(61, 0xa4506cebu) X(62, 0xbef9a3f7u) X(63, 0xc67178f2u)

// K[i] + W[i] for the padding block of a 64-byte message: W[0] = 0x80000000, W[1..14] = 0, W[15] = 512, W[16..63] its
// schedule.  tests/test_sha256_emulation.py recomputes them from K.
#define RONK_SHA256_KW_PAD64(X)                                                                                       \
  X(0, 0xc28a2f98u) X(1, 0x71374491u) X(2, 0xb5c0fbcfu) X(3, 0xe9b5dba5u)                                             \
  X(4, 0x3956c25bu) X(5, 0x59f111f1u) X(6, 0x923f82a4u) X(7, 0xab1c5ed5u)                                             \
  X(8, 0xd807aa98u) X(9, 0x12835b01u) X(10, 0x243185beu) X(11, 0x550c7dc3u)                                           \
  X(12, 0x72be5d74u) X(13, 0x80deb1feu) X(14, 0x9bdc06a7u) X(15, 0xc19bf374u)                                         \
  X(16, 0x649b69c1u) X(17, 0xf0fe4786u) X(18, 0x0fe1edc6u) X(19, 0x240cf254u)                                         \
  X(20, 0x4fe9346fu) X(21, 0x6cc984beu) X(22, 0x61b9411eu) X(23, 0x16f988fau)                                         \
  X(24, 0xf2c65152u) X(25, 0xa88e5a6du) X(26, 0xb019fc65u) X(27, 0xb9d99ec7u)                                         \
  X(28, 0x9a1231c3u) X(29, 0xe70eeaa0u) X(30, 0xfdb1232bu) X(31, 0xc7353eb0u)                                         \
  X(32, 0x3069bad5u) X(33, 0xcb976d5fu) X(34, 0x5a0f118fu) X(35, 0xdc1eeefdu)                                         \
  X(36, 0x0a35b689u) X(37, 0xde0b7a04u) X(38, 0x58f4ca9du) X(39, 0xe15d5b16u)                                         \
  X(40, 0x007f3e86u) X(41, 0x37088980u) X(42, 0xa507ea32u) X(43, 0x6fab9537u)                                         \
  X(44, 0x17406110u) X(45, 0x0d8cd6f1u) X(46, 0xcdaa3b6du) X(47, 0xc0bbbe37u)                                         \
  X(48, 0x83613bdau) X(49, 0xdb48a363u) X(50, 0x0b02e931u) X(51, 0x6fd15ca7u)                                         \
  X(52, 0x521afacau) X(53, 0x31338431u) X(54, 0x6ed41a95u) X(55, 0x6d437890u)                                         \
  X(56, 0xc39c91f2u) X(57, 0x9eccabbdu) X(58, 0xb5c9a0e6u) X(59, 0x532fb63cu)                                         \
  X(60, 0xd2c741c6u) X(61, 0x07237ea3u) X(62, 0xa4954b68u) X(63, 0x4c191d76u)

#define RONK_SHA256_CASE(i, v) case i: return v;
RONK_DEV constexpr u32 sha_k(int i) {
  switch (i) { RONK_SHA256_K(RONK_SHA256_CASE) }
  return 0;
}
RONK_DEV constexpr u32 sha_kw_pad64(int i) {
  switch (i) { RONK_SHA256_KW_PAD64(RONK_SHA256_CASE) }
  return 0;
}
#undef RONK_SHA256_CASE

// Initial hash value H(0) (FIPS 180-4 §5.3.3)
RONK_DEV void sha_init(u32 h[8]) {
  h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
  h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
}

RONK_DEV u32 sha_rotr(u32 x, int n) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_r(x, x, n);
#else
  return (x >> n) | (x << (32 - n));
#endif
}

// Bytes of the 8-byte value y:x picked by the four selector nibbles of s (CUDA's __byte_perm, selector values 0 … 7).
RONK_DEV u32 sha_byte_perm(u32 x, u32 y, u32 s) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(x, y, s);
#else
  const u64 v = ((u64)y << 32) | x;
  u32 r = 0;
  for (int i = 0; i < 4; i++) r |= (u32)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
  return r;
#endif
}

RONK_DEV u32 sha_bswap(u32 x) { return sha_byte_perm(x, 0, 0x0123); }

RONK_DEV u32 sha_S0(u32 a) { return sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22); }
RONK_DEV u32 sha_S1(u32 e) { return sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25); }
RONK_DEV u32 sha_s0(u32 w) { return sha_rotr(w, 7) ^ sha_rotr(w, 18) ^ (w >> 3); }
RONK_DEV u32 sha_s1(u32 w) { return sha_rotr(w, 17) ^ sha_rotr(w, 19) ^ (w >> 10); }
RONK_DEV u32 sha_ch(u32 e, u32 f, u32 g) { return (e & f) ^ (~e & g); }
RONK_DEV u32 sha_maj(u32 a, u32 b, u32 c) { return (a & b) ^ (a & c) ^ (b & c); }

// One round; kw = K[i] + W[i].  The caller rotates the names, so no register moves are emitted.
#define RONK_SHA256_ROUND(a, b, c, d, e, f, g, h, kw)              \
  do {                                                             \
    const u32 t1_ = h + sha_S1(e) + sha_ch(e, f, g) + (kw);        \
    d += t1_;                                                      \
    h = t1_ + sha_S0(a) + sha_maj(a, b, c);                        \
  } while (0)

// st ← st + compress(st, w): w holds the block's 16 big-endian words and is overwritten by the schedule window.
RONK_DEV void sha_compress(u32 st[8], u32 w[16]) {
  u32 a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int i = 0; i < 64; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int r = i + j;
      if (r >= 16) w[r & 15] += sha_s1(w[(r - 2) & 15]) + w[(r - 7) & 15] + sha_s0(w[(r - 15) & 15]);
    }
    RONK_SHA256_ROUND(a, b, c, d, e, f, g, h, sha_k(i + 0) + w[(i + 0) & 15]);
    RONK_SHA256_ROUND(h, a, b, c, d, e, f, g, sha_k(i + 1) + w[(i + 1) & 15]);
    RONK_SHA256_ROUND(g, h, a, b, c, d, e, f, sha_k(i + 2) + w[(i + 2) & 15]);
    RONK_SHA256_ROUND(f, g, h, a, b, c, d, e, sha_k(i + 3) + w[(i + 3) & 15]);
    RONK_SHA256_ROUND(e, f, g, h, a, b, c, d, sha_k(i + 4) + w[(i + 4) & 15]);
    RONK_SHA256_ROUND(d, e, f, g, h, a, b, c, sha_k(i + 5) + w[(i + 5) & 15]);
    RONK_SHA256_ROUND(c, d, e, f, g, h, a, b, sha_k(i + 6) + w[(i + 6) & 15]);
    RONK_SHA256_ROUND(b, c, d, e, f, g, h, a, sha_k(i + 7) + w[(i + 7) & 15]);
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// st ← st + compress(st, padding block of a 64-byte message): no schedule, K + W are immediates.
RONK_DEV void sha_compress_pad64(u32 st[8]) {
  u32 a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int i = 0; i < 64; i += 8) {
    RONK_SHA256_ROUND(a, b, c, d, e, f, g, h, sha_kw_pad64(i + 0));
    RONK_SHA256_ROUND(h, a, b, c, d, e, f, g, sha_kw_pad64(i + 1));
    RONK_SHA256_ROUND(g, h, a, b, c, d, e, f, sha_kw_pad64(i + 2));
    RONK_SHA256_ROUND(f, g, h, a, b, c, d, e, sha_kw_pad64(i + 3));
    RONK_SHA256_ROUND(e, f, g, h, a, b, c, d, sha_kw_pad64(i + 4));
    RONK_SHA256_ROUND(d, e, f, g, h, a, b, c, sha_kw_pad64(i + 5));
    RONK_SHA256_ROUND(c, d, e, f, g, h, a, b, sha_kw_pad64(i + 6));
    RONK_SHA256_ROUND(b, c, d, e, f, g, h, a, sha_kw_pad64(i + 7));
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}
#undef RONK_SHA256_ROUND

// The digest of the node L ‖ R (merkle.rs:44-50), all three as the eight big-endian words h0 … h7.
RONK_DEV void sha_node(const u32 l[8], const u32 r[8], u32 out[8]) {
  u32 w[16];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    w[i] = l[i];
    w[i + 8] = r[i];
  }
  sha_init(out);
  sha_compress(out, w);
  sha_compress_pad64(out);
}

// The little-endian aligned word at address a (a % 4 == 0) with the bytes outside [s, e) read as zero and never loaded.
RONK_DEV u32 sha_word_at(uintptr_t a, uintptr_t s, uintptr_t e) {
  if (a >= s && a + 4 <= e) return *(const u32*)a;
  u32 w = 0;
  for (int b = 0; b < 4; b++)
    if (a + b >= s && a + b < e) w |= (u32)*(const uint8_t*)(a + b) << (8 * b);
  return w;
}

// h = SHA-256 of the bytes [m, m + len), any alignment; only those bytes are read.  len < 2^61.
RONK_DEV void sha_message(const uint8_t* m, u64 len, u32 h[8]) {
  const uintptr_t s = (uintptr_t)m, e = s + len, sh = s & 3;
  const u32 sel = (u32)((sh << 12) | ((sh + 1) << 8) | ((sh + 2) << 4) | (sh + 3));
  const u64 blocks = (len + 8) / 64 + 1;
  const u64 bits = len * 8;
  uintptr_t a = s - sh;  // the aligned word that holds message byte 0
  u32 lo = sha_word_at(a, s, e);
  sha_init(h);
  for (u64 blk = 0; blk < blocks; blk++) {
    u32 w[16];
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const u64 q = blk * 64 + 4 * j;  // message offset of this word's first byte
      a += 4;
      const u32 hi = sha_word_at(a, s, e);
      u32 x = sha_byte_perm(lo, hi, sel);
      lo = hi;
      if (len >= q && len < q + 4) x |= 0x80000000u >> (8 * (len - q));
      w[j] = x;
    }
    if (blk + 1 == blocks) {
      w[14] = (u32)(bits >> 32);
      w[15] = (u32)bits;
    }
    sha_compress(h, w);
  }
}

// One node of the next level inside a span of a Merkle level held word-major: lvl[k·stride + i] is word k of node i,
// for the cnt nodes of this level in the span.  Node i of the next level hashes nodes 2i and 2i + 1; the span's last
// node, when cnt is odd, is paired with itself (merkle.rs:51-55) — only the span that holds the level's end has an odd
// count.  Reads 16 words, writes none.
RONK_DEV void merkle_span_node(const u32* lvl, u32 stride, u32 i, u32 cnt, u32 out[8]) {
  const u32 li = 2 * i, ri = 2 * i + 1 < cnt ? 2 * i + 1 : 2 * i;
  u32 l[8], r[8];
#pragma unroll
  for (int k = 0; k < 8; k++) {
    l[k] = lvl[k * stride + li];
    r[k] = lvl[k * stride + ri];
  }
  sha_node(l, r, out);
}

}  // namespace ronk
