/* A host WITHOUT Python: replays an exported UNet plan (gligen_b200/export.py) through the engine-level C ABI of
 * libgligen_b200.so (include/gligen_b200.h: glg_engine_*) - the stand-in for the cgo / JNI / N-API binding a non-Python
 * maintainer would write (INTEGRATION.md 3).
 *
 *   gcc -O2 -I include examples/host_c/unet_host.c -L gligen_b200 -lgligen_b200 -Wl,-rpath,$PWD/gligen_b200 -o unet_host
 *   ./unet_host plan.glgplan out.bin  name=file.bin ...      (each "name=file" fills the named input buffer from a raw file)
 *
 * Runs the static part once and the per-step part once on the default stream, writes the "out" buffer (fp32 eps) to out.bin.
 * No CUDA headers are needed: buffers are filled from pageable HOST memory by glg_engine_write and read back by glg_engine_read
 * (cudaMemcpyAsync with cudaMemcpyDefault underneath: for pageable host memory the call returns when the host side of the copy
 * is done, and everything here is ordered on the default stream). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gligen_b200.h"

static void die(const char* what) {
  fprintf(stderr, "unet_host: %s: %s\n", what, glg_last_error());
  exit(1);
}

static void* slurp(const char* path, long long* n) {
  FILE* f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "unet_host: cannot open %s\n", path); exit(1); }
  fseek(f, 0, SEEK_END);
  *n = ftell(f);
  fseek(f, 0, SEEK_SET);
  void* p = malloc((size_t)*n);
  if (fread(p, 1, (size_t)*n, f) != (size_t)*n) { fprintf(stderr, "unet_host: short read %s\n", path); exit(1); }
  fclose(f);
  return p;
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: %s plan.glgplan out.bin [name=file.bin ...] [fuser=0|1]\n", argv[0]); return 2; }
  if (glg_abi_version() != GLG_ABI_VERSION) { fprintf(stderr, "unet_host: header / library ABI mismatch\n"); return 1; }
  GlgEngine* e = NULL;
  if (glg_engine_load(argv[1], &e)) die(argv[1]);          /* a refused plan: the message names the op and what is wrong */
  int fuser_on = 1;
  for (int i = 3; i < argc; ++i) {
    char* eq = strchr(argv[i], '=');
    if (!eq) { fprintf(stderr, "unet_host: bad argument %s\n", argv[i]); return 2; }
    *eq = 0;
    if (!strcmp(argv[i], "fuser")) { fuser_on = atoi(eq + 1); continue; }
    long long n = 0, cap = 0;
    void* dev = NULL;
    void* host = slurp(eq + 1, &n);
    if (glg_engine_buffer(e, argv[i], &dev, (int64_t*)&cap)) die(argv[i]);
    if (n != cap) { fprintf(stderr, "unet_host: %s holds %lld bytes, buffer %s wants %lld\n", eq + 1, n, argv[i], cap); return 1; }
    if (glg_engine_write(e, argv[i], host, n, NULL)) die("glg_engine_write");
    free(host);
  }
  if (glg_engine_run(e, /*static_part=*/1, fuser_on, NULL)) die("glg_engine_run(static)");
  if (glg_engine_run(e, /*static_part=*/0, fuser_on, NULL)) die("glg_engine_run(step)");
  void* dev = NULL;
  long long nout = 0;
  if (glg_engine_buffer(e, "out", &dev, (int64_t*)&nout)) die("out");
  float* out = (float*)malloc((size_t)nout);
  if (glg_engine_read(e, "out", out, nout, NULL)) die("glg_engine_read");
  FILE* f = fopen(argv[2], "wb");
  fwrite(out, 1, (size_t)nout, f);
  fclose(f);
  double s = 0;
  for (long long i = 0; i < nout / 4; ++i) s += out[i];
  printf("unet_host: %lld ops, %lld output floats, sum %.6f, %lld kernel launches\n", (long long)glg_engine_num_ops(e), nout / 4, s,
         (long long)glg_launch_count());
  free(out);
  glg_engine_destroy(e);
  return 0;
}
