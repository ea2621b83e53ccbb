/* poseidon_oracle.c — TEST INFRASTRUCTURE: the reference's Poseidon permutation (src/hashes/poseidon/mod.rs:39-149)
 * and its sponge state machine (sponge.rs:71-294), restated in C from the reference's algorithm for any prime
 * p < 2^64 with __int128 products, independent of the library's kernels and field policies.  The sponge follows the
 * reference's absorb and squeeze branches literally, so a test can compare any split of the calls with the library's
 * one-shot rows.  Loaded by tests/poseidon_oracle.py; never linked into libronk_b200.so. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef unsigned __int128 u128;

typedef struct {
  u64 p, alpha;
  size_t width, num_f, num_p;
  const u64 *rc;   /* (num_f + num_p)·width, canonical */
  const u64 *mds;  /* width², row-major, canonical */
} cfg;

static u64 add(u64 a, u64 b, u64 p) { return (u64)(((u128)a + b) % p); }
static u64 mul(u64 a, u64 b, u64 p) { return (u64)(((u128)a * b) % p); }
/* Field::pow (prime/mod.rs:74-84): pow(0) = ONE, pow(1) = self, else pow(e/2)² (· self for odd e) */
static u64 fpow(u64 x, u64 e, u64 p) {
  if (e == 0) return 1 % p;
  if (e == 1) return x;
  const u64 h = fpow(x, e / 2, p);
  const u64 sq = mul(h, h, p);
  return (e & 1) ? mul(sq, x, p) : sq;
}

/* Poseidon::hash's rounds on a state of `width` words, in place (mod.rs:137-149) */
static void permute(const cfg *c, u64 *s) {
  u64 n[64];
  const size_t T = c->width, R = c->num_f + c->num_p;
  for (size_t i = 0; i < R; i++) {
    for (size_t k = 0; k < T; k++) s[k] = add(s[k], c->rc[i * T + k], c->p);   /* add_round_constants */
    if (i < c->num_f / 2 || i >= c->num_p + c->num_f / 2)                      /* apply_non_linear_layer */
      for (size_t k = 0; k < T; k++) s[k] = fpow(s[k], c->alpha, c->p);
    else
      s[0] = fpow(s[0], c->alpha, c->p);
    for (size_t r = 0; r < T; r++) {                                           /* apply_linear_layer */
      u64 acc = 0;
      for (size_t j = 0; j < T; j++) acc = add(acc, mul(s[j], c->mds[r * T + j], c->p), c->p);
      n[r] = acc;
    }
    memcpy(s, n, T * sizeof(u64));
  }
}

void orc_pos_permute(u64 p, size_t width, u64 alpha, size_t num_f, size_t num_p, const u64 *rc, const u64 *mds, u64 *states,
                     size_t batch) {
  const cfg c = {p, alpha, width, num_f, num_p, rc, mds};
  for (size_t y = 0; y < batch; y++) permute(&c, states + y * width);
}

/* PoseidonSponge's fields (sponge.rs:71-100) */
typedef struct {
  cfg c;
  u64 state[64];
  size_t rate, capacity, absorb_index, squeeze_index;
} sponge;

static void sp_permute(sponge *s) { permute(&s->c, s->state); s->absorb_index = 0; }  /* sponge.rs:103-107 */

/* absorb (sponge.rs:142-194) */
static void sp_absorb(sponge *s, const u64 *e, size_t n) {
  const u64 p = s->c.p;
  if (s->absorb_index + n <= s->rate) {
    for (size_t i = 0; i < n; i++) s->state[s->capacity + s->absorb_index + i] = add(s->state[s->capacity + s->absorb_index + i], e[i], p);
    s->absorb_index += n;
    return;
  } else if (s->absorb_index != 0) {
    const size_t take = s->rate - s->absorb_index;
    for (size_t i = 0; i < take; i++) s->state[s->capacity + s->absorb_index + i] = add(s->state[s->capacity + s->absorb_index + i], e[i], p);
    e += take;
    n -= take;
    sp_permute(s);
  }
  const size_t chunks = n / s->rate;
  for (size_t k = 0; k < chunks; k++) {
    for (size_t i = 0; i < s->rate; i++)
      s->state[s->capacity + s->absorb_index + i] = add(s->state[s->capacity + s->absorb_index + i], e[k * s->rate + i], p);
    sp_permute(s);
  }
  const size_t rem = n - chunks * s->rate;
  if (rem) {
    for (size_t i = 0; i < rem; i++) s->state[s->capacity + i] = add(s->state[s->capacity + i], e[chunks * s->rate + i], p);
    s->absorb_index = rem;
  }
}

/* start_squeezing (sponge.rs:198-213) */
static void sp_start_squeezing(sponge *s) {
  if (s->absorb_index != 0) sp_permute(s);
}

/* squeeze (sponge.rs:244-274) */
static void sp_squeeze(sponge *s, u64 *out, size_t n) {
  size_t taken = 0;
  for (;;) {
    const size_t left = n - taken;
    if (s->squeeze_index + left <= s->rate) {
      memcpy(out + taken, s->state + s->capacity + s->squeeze_index, left * sizeof(u64));
      s->squeeze_index += left;
      return;
    }
    const size_t size = left < s->rate - s->squeeze_index ? left : s->rate - s->squeeze_index;
    memcpy(out + taken, s->state + s->capacity + s->squeeze_index, size * sizeof(u64));
    s->squeeze_index += size;
    if (s->squeeze_index == s->rate) {
      sp_permute(s);
      s->squeeze_index = 0;
    }
    taken += size;
  }
}

/* One fresh sponge (PoseidonSponge::new, start_absorbing) that absorbs `in` in n_abs calls of abs[k] words, starts
 * squeezing and squeezes n_sq calls of sq[k] words into out (Σ sq words).  Returns 1 where the reference panics or
 * never returns (width < 2 is PoseidonConfig::new's assert; rate == 0 or rate > width). */
int orc_pos_sponge(u64 p, size_t width, u64 alpha, size_t num_f, size_t num_p, const u64 *rc, const u64 *mds, size_t rate,
                   const u64 *in, const size_t *abs, size_t n_abs, const size_t *sq, size_t n_sq, u64 *out) {
  if (width < 2 || width > 64 || rate == 0 || rate > width) return 1;
  sponge s;
  memset(&s, 0, sizeof(s));
  s.c = (cfg){p, alpha, width, num_f, num_p, rc, mds};
  s.rate = rate;
  s.capacity = width - rate;
  for (size_t k = 0; k < n_abs; k++) {
    sp_absorb(&s, in, abs[k]);
    in += abs[k];
  }
  sp_start_squeezing(&s);
  for (size_t k = 0; k < n_sq; k++) {
    sp_squeeze(&s, out, sq[k]);
    out += sq[k];
  }
  return 0;
}
