// TEST INFRASTRUCTURE: the device's ZSTD block routine (tikv_b200/csrc/zstd_block.h) built for the CPU with one lane and
// a heap workspace, run over a corpus of block contents under AddressSanitizer.  Every input and output lives in an
// allocation of exactly its size, so a read or a write the routine's checks let through aborts the run.
//
//   zstd_block_emul <corpus> <verdicts>
//   corpus   := (u32 LE n | n bytes of block contents: varint32 size | ZSTD frame)*
//   verdicts := (u8 verdict | u32 LE size | size bytes when verdict == 0)*
//               verdict 0 decoded, 1 corrupt (frame() or inflate()), 2 unsupported (frame(): no magic, a dictionary)
#include <cstdio>
#include <cstdlib>

#include "../tikv_b200/csrc/zstd_block.h"

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s corpus verdicts\n", argv[0]); return 2; }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) { perror("open"); return 2; }
  b2zstd::Workspace* ws = (b2zstd::Workspace*)malloc(sizeof(b2zstd::Workspace));
  uint32_t n;
  while (fread(&n, 4, 1, in) == 1) {
    uint8_t* src = (uint8_t*)malloc(n);
    if (fread(src, 1, n, in) != n) { fprintf(stderr, "truncated corpus\n"); return 2; }
    b2zstd::Frame f;
    uint8_t verdict = (uint8_t)b2zstd::frame(src, n, &f);
    uint8_t* dst = nullptr;
    if (verdict == b2zstd::kOk) {
      dst = (uint8_t*)malloc(f.size);
      if (!b2zstd::inflate(src, n, f, dst, ws, 0, 1)) verdict = b2zstd::kCorrupt;
    }
    const uint32_t out_size = verdict == b2zstd::kOk ? f.size : 0;
    fwrite(&verdict, 1, 1, out);
    fwrite(&out_size, 4, 1, out);
    if (out_size) fwrite(dst, 1, out_size, out);
    free(dst);
    free(src);
  }
  free(ws);
  fclose(in);
  fclose(out);
  return 0;
}
