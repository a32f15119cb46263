// TEST INFRASTRUCTURE: the device's LZ4 block routine (tikv_b200/csrc/lz4_block.h) built for the CPU with one lane, run
// over a corpus of block contents under AddressSanitizer.  Every input and output lives in an allocation of exactly its
// size, so a read or a write the routine's checks let through aborts the run.
//
//   lz4_block_emul <corpus> <verdicts>
//   corpus   := (u32 LE n | n bytes of block contents: varint32 size | LZ4 block)*
//   verdicts := (u8 ok | u32 LE size | size bytes when ok)*          ok = 0: rejected by frame() or inflate()
#include <cstdio>
#include <cstdlib>

#include "../tikv_b200/csrc/lz4_block.h"

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s corpus verdicts\n", argv[0]); return 2; }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) { perror("open"); return 2; }
  uint32_t n;
  while (fread(&n, 4, 1, in) == 1) {
    uint8_t* src = (uint8_t*)malloc(n);
    if (fread(src, 1, n, in) != n) { fprintf(stderr, "truncated corpus\n"); return 2; }
    uint32_t size = 0, at = 0;
    uint8_t ok = b2lz4::frame(src, n, &size, &at);
    uint8_t* dst = nullptr;
    if (ok) {
      dst = (uint8_t*)malloc(size);
      ok = b2lz4::inflate(src + at, n - at, dst, size, 0, 1);
    }
    const uint32_t out_size = ok ? size : 0;
    fwrite(&ok, 1, 1, out);
    fwrite(&out_size, 4, 1, out);
    if (ok) fwrite(dst, 1, size, out);
    free(dst);
    free(src);
  }
  fclose(in);
  fclose(out);
  return 0;
}
