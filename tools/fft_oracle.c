/* ORACLE -- test infrastructure, NOT product code: oracle_fft, the scalar-field FFT checker of tests/test_fft*.py and the CPU arm of
 * tools/bench_fft.py. It restates the reference's iterative loops (constantine/math/polynomials/fft_fields.nim:156-340: DIF natural
 * -> bit-reversed, DIT bit-reversed -> natural with the reversed root table and the 1/n factor; :532-740 the eight entries with
 * shift_vals / unshift_vals) over the runtime field_t and Montgomery multiplication of the MSM oracle, which it compiles in unchanged
 * (oracle/msm_oracle.c). Threaded over the butterflies of a stage across the whole batch, and over the elements of the scaling steps.
 *
 * Build: gcc -O3 -march=x86-64-v3 -fPIC -pthread -shared -o tools/bin/libfft_oracle.so tools/fft_oracle.c (done by build()).
 */
#include "../oracle/msm_oracle.c"

typedef fp_4_1 fr_t;   /* every scalar field here is 4 x u64 */

static void fr_one(fr_t* r, const field_t* f) { for (int i = 0; i < 4; i++) r->l[i] = f->one[i]; }
static void fr_pow(fr_t* r, const fr_t* a, uint64_t e, const field_t* f) {
  fr_t acc, b = *a;
  fr_one(&acc, f);
  for (; e; e >>= 1) {
    if (e & 1) fp_mul_4_1(&acc, &acc, &b, f);
    fp_mul_4_1(&b, &b, &b, f);
  }
  *r = acc;
}

/* ---- a minimal parallel for: [0, count) split into nthreads contiguous ranges ---- */
typedef void (*range_fn)(void* ctx, size_t lo, size_t hi);
typedef struct { range_fn fn; void* ctx; size_t lo, hi; } range_task;
static void* range_run(void* a) { range_task* t = (range_task*)a; t->fn(t->ctx, t->lo, t->hi); return NULL; }
static void parallel_for(size_t count, int nthreads, range_fn fn, void* ctx) {
  if (nthreads < 1) nthreads = 1;
  if ((size_t)nthreads > count / 4096 + 1) nthreads = (int)(count / 4096 + 1);
  if (nthreads == 1) { fn(ctx, 0, count); return; }
  pthread_t th[256];
  range_task tk[256];
  if (nthreads > 256) nthreads = 256;
  for (int i = 0; i < nthreads; i++) {
    tk[i].fn = fn; tk[i].ctx = ctx;
    tk[i].lo = count * i / nthreads; tk[i].hi = count * (i + 1) / nthreads;
    pthread_create(&th[i], NULL, range_run, &tk[i]);
  }
  for (int i = 0; i < nthreads; i++) pthread_join(th[i], NULL);
}

typedef struct {
  const field_t* f;
  fr_t* v;              /* batch x n */
  const fr_t* v_in;
  fr_t* tmp;
  size_t n;
  int log_n;
  const fr_t* roots;    /* rootz of the stage loop: roots[k] = w_n^(+-k), k < n/2 */
  size_t length;        /* current butterfly group length */
  fr_t x;               /* per-element factor base: coset shift or its inverse */
  fr_t scale;
} fft_ctx;

/* reference fft_nr_impl_iterative_dif, one `length` level: out[i+j] += out[i+j+half]; out[i+j+half] = (a - b) * roots[j*step] */
static void dif_level(void* c_, size_t lo, size_t hi) {
  fft_ctx* c = (fft_ctx*)c_;
  const size_t n = c->n, half = c->length >> 1, step = n / c->length;
  for (size_t b = lo; b < hi; b++) {
    const size_t t = b / (n / 2), bb = b % (n / 2);
    const size_t i = t * n + (bb / half) * c->length, j = bb % half;
    fr_t* x = &c->v[i + j];
    fr_t* y = &c->v[i + j + half];
    fr_t d;
    fp_sub_4_1(&d, x, y, c->f);
    fp_add_4_1(x, x, y, c->f);
    fp_mul_4_1(y, &d, &c->roots[j * step], c->f);
  }
}

/* reference fft_rn_impl_iterative_dit / ifft_rn_impl_iterative_dit, one level: t = out[i+j+half] * roots[j*step] */
static void dit_level(void* c_, size_t lo, size_t hi) {
  fft_ctx* c = (fft_ctx*)c_;
  const size_t n = c->n, half = c->length >> 1, step = n / c->length;
  for (size_t b = lo; b < hi; b++) {
    const size_t t = b / (n / 2), bb = b % (n / 2);
    const size_t i = t * n + (bb / half) * c->length, j = bb % half;
    fr_t* x = &c->v[i + j];
    fr_t* y = &c->v[i + j + half];
    fr_t m;
    fp_mul_4_1(&m, y, &c->roots[j * step], c->f);
    fp_sub_4_1(y, x, &m, c->f);
    fp_add_4_1(x, x, &m, c->f);
  }
}

/* out[i] *= scale * x^(i mod n) (shift_vals / unshift_vals and the 1/n factor); each range starts from x^i by exponentiation */
static void scale_range(void* c_, size_t lo, size_t hi) {
  fft_ctx* c = (fft_ctx*)c_;
  fr_t p;
  fr_pow(&p, &c->x, lo % c->n, c->f);
  for (size_t e = lo; e < hi; e++) {
    if (e % c->n == 0) fr_one(&p, c->f);
    fr_t s;
    fp_mul_4_1(&s, &p, &c->scale, c->f);
    fp_mul_4_1(&c->v[e], &c->v[e], &s, c->f);
    fp_mul_4_1(&p, &p, &c->x, c->f);
  }
}

static size_t brev_sz(size_t i, int bits) {
  size_t r = 0;
  for (int b = 0; b < bits; b++) r |= ((i >> b) & 1) << (bits - 1 - b);
  return r;
}
static void gather_brev(void* c_, size_t lo, size_t hi) {
  fft_ctx* c = (fft_ctx*)c_;
  for (size_t e = lo; e < hi; e++) {
    const size_t base = e - e % c->n;
    c->tmp[e] = c->v_in[base + brev_sz(e % c->n, c->log_n)];
  }
}
static void copy_range(void* c_, size_t lo, size_t hi) {
  fft_ctx* c = (fft_ctx*)c_;
  memcpy(&c->v[lo], &c->tmp[lo], (hi - lo) * sizeof(fr_t));
}

static void bit_reverse(fft_ctx* c, size_t total, int nthreads) {
  c->v_in = c->v;
  c->tmp = (fr_t*)malloc(total * sizeof(fr_t));
  parallel_for(total, nthreads, gather_brev, c);
  parallel_for(total, nthreads, copy_range, c);
  free(c->tmp);
}

/* kinds: 0 fft_nn, 1 fft_nr, 2 ifft_nn, 3 ifft_rn, 4 coset_fft_nn, 5 coset_fft_nr, 6 coset_ifft_nn, 7 coset_ifft_rn.
 * omega: the domain's generator (Montgomery), of order 2^log_order; shift: the coset shift (Montgomery), kinds 4..7.
 * Returns the reference's FFTStatus: 2 n > N, 3 n not a power of two (n = 0 included), else 0 with out written. out may be in. */
int oracle_fft(const field_t* f, int kind, uint64_t* out, const uint64_t* in, size_t n, size_t batch, const uint64_t* omega,
               int log_order, const uint64_t* shift, int nthreads) {
  if (n > ((size_t)1 << log_order)) return 2;
  if (n == 0 || (n & (n - 1))) return 3;
  const size_t total = n * batch;
  if (out != in) memmove(out, in, total * sizeof(fr_t));
  if (total == 0) return 0;
  int log_n = 0;
  while (((size_t)1 << log_n) < n) log_n++;
  const int inverse = kind == 2 || kind == 3 || kind == 6 || kind == 7;
  const int nn = kind == 0 || kind == 2 || kind == 4 || kind == 6;
  const int coset = kind >= 4;
  fft_ctx c;
  memset(&c, 0, sizeof c);
  c.f = f; c.v = (fr_t*)out; c.n = n; c.log_n = log_n;
  /* the strided root table: w_n = omega^(N/n); the inverse reads the reversed table, w_n^(-k) = w_n^(n-k) */
  fr_t w;
  memcpy(&w, omega, sizeof w);
  for (int i = log_n; i < log_order; i++) fp_mul_4_1(&w, &w, &w, f);
  if (inverse) fr_pow(&w, &w, n - 1, f);
  fr_t* roots = (fr_t*)malloc((n / 2 + 1) * sizeof(fr_t));
  fr_one(&roots[0], f);
  for (size_t k = 1; k < n / 2; k++) fp_mul_4_1(&roots[k], &roots[k - 1], &w, f);
  c.roots = roots;
  if (coset && !inverse) {                               /* shift_vals */
    memcpy(&c.x, shift, sizeof c.x);
    fr_one(&c.scale, f);
    parallel_for(total, nthreads, scale_range, &c);
  }
  if (!inverse) {
    for (c.length = n; c.length >= 2; c.length >>= 1) parallel_for(total / 2, nthreads, dif_level, &c);
    if (nn) bit_reverse(&c, total, nthreads);
  } else {
    if (nn) bit_reverse(&c, total, nthreads);          /* ifft_nn_via_bitrev_and_iterative_dit */
    for (c.length = 2; c.length <= n; c.length <<= 1) parallel_for(total / 2, nthreads, dit_level, &c);
    fr_t nm;                                            /* invLen.fromUint(n); inv_vartime */
    fr_one(&nm, f);
    for (int i = 0; i < log_n; i++) fp_add_4_1(&nm, &nm, &nm, f);
    fp_inv_4_1(&c.scale, &nm, f);
    if (coset) {                                       /* unshift_vals with inv_vartime(cosetShift) */
      fr_t g;
      memcpy(&g, shift, sizeof g);
      fp_inv_4_1(&c.x, &g, f);
    } else {
      fr_one(&c.x, f);
    }
    parallel_for(total, nthreads, scale_range, &c);
  }
  free(roots);
  return 0;
}

/* sum_j a_j x^j over n residues, threaded over chunks (each chunk starts from x^lo): one output of a transform in O(n) */
typedef struct { const field_t* f; const fr_t* a; fr_t x; fr_t part[256]; size_t chunk; } eval_ctx;
static void eval_range(void* c_, size_t lo, size_t hi) {
  eval_ctx* c = (eval_ctx*)c_;
  fr_t p, acc, t;
  fr_pow(&p, &c->x, lo, c->f);
  memset(&acc, 0, sizeof acc);
  for (size_t j = lo; j < hi; j++) {
    fp_mul_4_1(&t, &c->a[j], &p, c->f);
    fp_add_4_1(&acc, &acc, &t, c->f);
    fp_mul_4_1(&p, &p, &c->x, c->f);
  }
  c->part[lo / c->chunk] = acc;
}
void oracle_fft_eval(const field_t* f, uint64_t* out, const uint64_t* a, size_t n, const uint64_t* x, int nthreads) {
  if (nthreads < 1) nthreads = 1;
  if (nthreads > 256) nthreads = 256;
  eval_ctx* c = (eval_ctx*)calloc(1, sizeof(eval_ctx));
  c->f = f; c->a = (const fr_t*)a;
  memcpy(&c->x, x, sizeof c->x);
  c->chunk = (n + nthreads - 1) / nthreads;
  if (c->chunk == 0) c->chunk = 1;
  const size_t parts = (n + c->chunk - 1) / c->chunk;
  pthread_t th[256];
  range_task tk[256];
  for (size_t i = 0; i < parts; i++) {
    tk[i].fn = eval_range; tk[i].ctx = c;
    tk[i].lo = i * c->chunk; tk[i].hi = (i + 1) * c->chunk < n ? (i + 1) * c->chunk : n;
    pthread_create(&th[i], NULL, range_run, &tk[i]);
  }
  fr_t acc;
  memset(&acc, 0, sizeof acc);
  for (size_t i = 0; i < parts; i++) {
    pthread_join(th[i], NULL);
    fp_add_4_1(&acc, &acc, &c->part[i], f);
  }
  memcpy(out, &acc, sizeof acc);
  free(c);
}
