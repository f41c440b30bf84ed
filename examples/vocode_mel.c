/* vocode_mel.c -- vocode mel spectrograms through the C ABI alone: include/wavernn_b200.h, libwavernn_b200.so and
 * libc; no Python, no PyTorch.  Built by wavernn_b200/csrc/Makefile into wavernn_b200/wrnn_vocode_mel.
 *
 *   wrnn_vocode_mel WEIGHTS_DIR MEL OUT [MEL OUT ...] [name=value ...]
 *
 * One MEL OUT pair is vocoded with wrnn_vocode_host.  Several pairs are vocoded as one batch with wrnn_vocode_many_host,
 * utterance i keyed by seed + i (each waveform is then what a single call with that seed gives on the same engine).
 * The options are the arguments that contain '=' (so a MEL or OUT path must not).
 *
 * WEIGHTS_DIR holds one raw little-endian float32 file per state_dict key, named "<key>.f32" (INTEGRATION.md section 2:
 * `for k, v in sd.items(): v.float().numpy().astype('<f4').tofile(f'{dir}/{k}.f32')`).  MEL is raw float32 [80, T],
 * the layout of the reference's mel .npy; OUT receives the float64 waveform of (T-1)*275 samples.
 * Options (defaults = the reference's hparams): mode=MOL|RAW (RAW: 9 bits), precision=fp16|bf16|fp32,
 * engine=auto|simt|tcgen05|stream, batched=1, target=11000, overlap=550, mu_law=1, seed=0, res_blocks=10, device=0. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "wavernn_b200.h"

#define MAX_KEYS 256

static const char *HOT_KEYS[16] = {"I.weight", "I.bias",
                                   "rnn1.weight_ih_l0", "rnn1.weight_hh_l0", "rnn1.bias_ih_l0", "rnn1.bias_hh_l0",
                                   "rnn2.weight_ih_l0", "rnn2.weight_hh_l0", "rnn2.bias_ih_l0", "rnn2.bias_hh_l0",
                                   "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"};

static float *read_f32(const char *path, int64_t *numel) {
  FILE *f = fopen(path, "rb");
  if (!f) { fprintf(stderr, "cannot open %s\n", path); return NULL; }
  fseek(f, 0, SEEK_END);
  long bytes = ftell(f);
  fseek(f, 0, SEEK_SET);
  float *p = bytes > 0 ? malloc((size_t)bytes) : NULL;
  if (!p || bytes % 4 || fread(p, 1, (size_t)bytes, f) != (size_t)bytes) {
    fprintf(stderr, "cannot read %s\n", path);
    free(p); fclose(f);
    return NULL;
  }
  fclose(f);
  *numel = bytes / 4;
  return p;
}

static int load_key(const char *dir, const char *key, wrnn_tensor *t) {
  char path[4096];
  snprintf(path, sizeof path, "%s/%s.f32", dir, key);
  t->name = key;
  t->data = read_f32(path, &t->numel);
  return t->data ? 0 : -1;
}

static int first_opt = 2;            /* index of the first name=value argument */

static const char *opt(int argc, char **argv, const char *name, const char *dflt) {
  size_t n = strlen(name);
  for (int i = first_opt; i < argc; ++i)
    if (!strncmp(argv[i], name, n) && argv[i][n] == '=') return argv[i] + n + 1;
  return dflt;
}

int main(int argc, char **argv) {
  while (first_opt < argc && !strchr(argv[first_opt], '=')) ++first_opt;
  const int n_utts = (first_opt - 2) / 2;
  if (n_utts < 1 || (first_opt - 2) % 2) {
    fprintf(stderr, "usage: %s WEIGHTS_DIR MEL OUT [MEL OUT ...] [name=value ...]\n", argv[0]);
    return 2;
  }
  const char *dir = argv[1];
  const int raw = !strcmp(opt(argc, argv, "mode", "MOL"), "RAW");
  const char *prec = opt(argc, argv, "precision", "fp16"), *eng = opt(argc, argv, "engine", "auto");
  const int res_blocks = atoi(opt(argc, argv, "res_blocks", "10"));

  /* the 16 tensors of the sample loop */
  static char names[MAX_KEYS][128];
  static wrnn_tensor t[MAX_KEYS];
  const float *hot[16];
  int n = 0, rc;
  for (int i = 0; i < 16; ++i) {
    if (load_key(dir, HOT_KEYS[i], &t[n])) return 1;
    hot[i] = t[n++].data;
  }
  wrnn_weights w = {hot[0], hot[1], hot[2], hot[3], hot[4], hot[5], hot[6], hot[7],
                    hot[8], hot[9], hot[10], hot[11], hot[12], hot[13], hot[14], hot[15]};
  wrnn_cfg cfg = {512, 512, 80, 32, raw ? 512 : 30, raw ? WRNN_MODE_RAW : WRNN_MODE_MOL,
                  !strcmp(prec, "fp32") ? WRNN_PREC_FP32 : !strcmp(prec, "bf16") ? WRNN_PREC_BF16 : WRNN_PREC_F16,
                  !strcmp(eng, "simt") ? WRNN_ENGINE_SIMT : !strcmp(eng, "tcgen05") ? WRNN_ENGINE_TCGEN05
                  : !strcmp(eng, "stream") ? WRNN_ENGINE_STREAM : WRNN_ENGINE_AUTO};
  wrnn_t *h = NULL;
  if ((rc = wrnn_create(&h, &cfg, &w, atoi(opt(argc, argv, "device", "0")))) != WRNN_OK) {
    fprintf(stderr, "wrnn_create: %d %s\n", rc, wrnn_last_error());
    return 1;
  }

  /* the conditioning network: upsample.* */
  const int first_up = n;
  const char *bn[4] = {"weight", "bias", "running_mean", "running_var"};
  snprintf(names[n], 128, "upsample.resnet.conv_in.weight"); ++n;
  for (int s = 0; s < 4; ++s) { snprintf(names[n], 128, "upsample.resnet.batch_norm.%s", bn[s]); ++n; }
  for (int r = 0; r < res_blocks && n + 12 < MAX_KEYS; ++r) {
    snprintf(names[n++], 128, "upsample.resnet.layers.%d.conv1.weight", r);
    snprintf(names[n++], 128, "upsample.resnet.layers.%d.conv2.weight", r);
    for (int s = 0; s < 4; ++s) snprintf(names[n++], 128, "upsample.resnet.layers.%d.batch_norm1.%s", r, bn[s]);
    for (int s = 0; s < 4; ++s) snprintf(names[n++], 128, "upsample.resnet.layers.%d.batch_norm2.%s", r, bn[s]);
  }
  snprintf(names[n++], 128, "upsample.resnet.conv_out.weight");
  snprintf(names[n++], 128, "upsample.resnet.conv_out.bias");
  for (int i = 0; i < 3; ++i) snprintf(names[n++], 128, "upsample.up_layers.%d.weight", 2 * i + 1);
  for (int i = first_up; i < n; ++i)
    if (load_key(dir, names[i], &t[i])) return 1;
  wrnn_upsample_cfg ucfg = {128, 128, res_blocks, 2, 3, {5, 5, 11, 0}, 275};
  if ((rc = wrnn_attach_upsampler(h, &ucfg, t, n)) != WRNN_OK) {
    fprintf(stderr, "wrnn_attach_upsampler: %d %s\n", rc, wrnn_last_error());
    return 1;
  }

  const int batched = atoi(opt(argc, argv, "batched", "1")), target = atoi(opt(argc, argv, "target", "11000"));
  const int overlap = atoi(opt(argc, argv, "overlap", "550")), mu_law = atoi(opt(argc, argv, "mu_law", "1"));
  const uint64_t seed = strtoull(opt(argc, argv, "seed", "0"), NULL, 10);
  wrnn_utterance *u = calloc((size_t)n_utts, sizeof(wrnn_utterance));
  if (!u) { fprintf(stderr, "out of memory\n"); return 1; }
  for (int i = 0; i < n_utts; ++i) {
    int64_t mel_numel = 0;
    float *mel = read_f32(argv[2 + 2 * i], &mel_numel);
    if (!mel || mel_numel % 80) { fprintf(stderr, "the mel file %s must hold [80, T] float32\n", argv[2 + 2 * i]); return 1; }
    const int64_t T = mel_numel / 80, wave_len = (T - 1) * 275;
    u[i].mel = mel;
    u[i].T = T;
    u[i].philox_seed = seed + (uint64_t)i;
    u[i].wav = malloc((size_t)(wave_len > 0 ? wave_len : 1) * sizeof(double));
  }
  if (n_utts == 1) {
    wrnn_vocode_job job = {u[0].mel, u[0].T, batched, target, overlap, mu_law, seed, u[0].wav};
    if ((rc = wrnn_vocode_host(h, &job)) != WRNN_OK) {
      fprintf(stderr, "wrnn_vocode_host: %d %s\n", rc, wrnn_last_error());
      return 1;
    }
  } else {
    wrnn_vocode_batch b = {u, n_utts, batched, target, overlap, mu_law};
    if ((rc = wrnn_vocode_many_host(h, &b)) != WRNN_OK) {
      fprintf(stderr, "wrnn_vocode_many_host: %d %s\n", rc, wrnn_last_error());
      return 1;
    }
  }
  for (int i = 0; i < n_utts; ++i) {
    const int64_t wave_len = (u[i].T - 1) * 275;
    const char *out = argv[3 + 2 * i];
    FILE *f = fopen(out, "wb");
    if (!f || fwrite(u[i].wav, sizeof(double), (size_t)wave_len, f) != (size_t)wave_len) { fprintf(stderr, "cannot write %s\n", out); return 1; }
    fclose(f);
    printf("%lld samples (%s engine)\n", (long long)wave_len, wrnn_engine_name(h));
  }
  wrnn_destroy(h);
  for (int i = 0; i < n; ++i) free((void *)t[i].data);
  for (int i = 0; i < n_utts; ++i) { free((void *)u[i].mel); free(u[i].wav); }
  free(u);
  return 0;
}
