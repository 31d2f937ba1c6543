/*
 * ref_emit.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The reference's own bytes for single deflate blocks.  AddLZ77Block, EncodeTree and the code-length
 * choice they rest on are `static` in deflate.c, so unlike ref_seams.c (which only CALLS the reference),
 * this TU COMPILES the reference's deflate.c IN PLACE: the #include below names the file where it lies
 * under $(REF)/src/zopfli at build time; nothing of it is copied into this repository.  oracle/Makefile
 * builds it into _ref/libref_emit.so with every symbol hidden except the two wrappers below, and links
 * it against _ref/libzopfli_ref.so for the reference's other translation units.
 */
#include "deflate.c"

#define REF_EMIT_API __attribute__((visibility("default")))

/* AddLZ77Block (deflate.c:682-745) for pieces i = 0..npieces-1 of one LZ77 store, one after the other:
 * symbols [lstart[i], lend[i]) of (litlens, dists), block type btype[i] (0 stored, 1 fixed, 2 dynamic),
 * BFINAL final[i].  The store's first symbol covers in[0].  The output starts at bit bp0 (0..7) of a
 * one-byte buffer holding 0 (bp0 == 0: an empty buffer), as when a caller's stream ends there.  Copies
 * the whole buffer to dst when it fits in cap bytes; returns its size and the final bit pointer. */
REF_EMIT_API size_t ref_emit_blocks(const unsigned char* in, const unsigned short* litlens,
                                    const unsigned short* dists, size_t n, size_t npieces,
                                    const size_t* lstart, const size_t* lend, const int* btype,
                                    const int* final, int bp0, unsigned char* dst, size_t cap,
                                    unsigned char* bp_out) {
  ZopfliOptions options;
  ZopfliLZ77Store store;
  unsigned char* out = 0;
  size_t outsize = 0, i, pos = 0;
  unsigned char bp = (unsigned char)bp0;
  ZopfliInitOptions(&options);
  ZopfliInitLZ77Store(in, &store);
  for (i = 0; i < n; i++) {
    ZopfliStoreLitLenDist(litlens[i], dists[i], pos, &store);
    pos += dists[i] == 0 ? 1 : litlens[i];
  }
  if (bp0) ZOPFLI_APPEND_DATA(0, &out, &outsize);
  for (i = 0; i < npieces; i++) {
    AddLZ77Block(&options, btype[i], final[i], &store, lstart[i], lend[i], 0, &bp, &out, &outsize);
  }
  if (outsize <= cap) memcpy(dst, out, outsize);
  *bp_out = bp;
  free(out);
  ZopfliCleanLZ77Store(&store);
  return outsize;
}

/* EncodeTree (deflate.c:105-249) of 288 + 32 code lengths with flags use_16 | use_17 << 1 | use_18 << 2:
 * returns the size in bits; with dst non-NULL also writes the encoding from bit 0 (at most cap bytes). */
REF_EMIT_API size_t ref_encode_tree(const unsigned* ll_lengths, const unsigned* d_lengths, int flags,
                                    unsigned char* dst, size_t cap) {
  unsigned char bp = 0;
  unsigned char* out = 0;
  size_t outsize = 0, bits;
  if (!dst) return EncodeTree(ll_lengths, d_lengths, flags & 1, flags & 2, flags & 4, 0, 0, 0);
  bits = EncodeTree(ll_lengths, d_lengths, flags & 1, flags & 2, flags & 4, &bp, &out, &outsize);
  if (outsize <= cap) memcpy(dst, out, outsize);
  free(out);
  return bits;
}
