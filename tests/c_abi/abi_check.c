/* Plain-C consumer of include/issue_emb_b200.h: proves the header is valid C (no C++-isms), that every entry point
 * links from libissue_emb_b200.so, and -- on a box without a GPU -- that creation fails with an error code and a message
 * instead of aborting or falling back to the CPU.  Built and run by tests/test_host_logic.py. */
#include <stdio.h>
#include <string.h>

#include "issue_emb_b200.h"

int main(void) {
  ie_config cfg;
  ie_encoder* enc = NULL;
  ie_mlp* mlp = NULL;
  int32_t dims[3] = {8, 4, 2};
  int rc;
  /* take the address of every declared function so that a missing export is a link error */
  typedef void (*fn)(void);
  fn syms[] = {(fn)ie_version, (fn)ie_last_error, (fn)ie_encoder_create, (fn)ie_encoder_destroy,
               (fn)ie_encoder_load_embedding, (fn)ie_encoder_load_layer, (fn)ie_encoder_encode, (fn)ie_encoder_raw_features,
               (fn)ie_encoder_launch_count, (fn)ie_encoder_max_batch, (fn)ie_encoder_last_phase_ms, (fn)ie_debug_seq_trace,
               (fn)ie_debug_workspace_bytes,
               (fn)ie_encoder_check_errors, (fn)ie_encoder_last_phase_mhz, (fn)ie_mlp_create, (fn)ie_mlp_load_layer, (fn)ie_mlp_predict_proba,
               (fn)ie_mlp_destroy, (fn)ie_pr_thresholds, (fn)ie_debug_gemm, (fn)ie_debug_gemm_ex,
               (fn)ie_debug_layer_states, (fn)ie_debug_gates};
  memset(&cfg, 0, sizeof cfg);
  cfg.n_layers = 4; cfg.emb_sz = 800; cfg.n_hid = 2400; cfg.vocab_sz = 60000; cfg.pad_idx = 1;
  printf("version=%d symbols=%d max_batch=%d\n", ie_version(), (int)(sizeof syms / sizeof syms[0]), IE_MAX_BATCH);
  rc = ie_encoder_create(NULL, &enc);
  printf("create(NULL)=%d msg=%s\n", rc, ie_last_error());
  if (rc != IE_ERR_INVALID) return 2;
  rc = ie_encoder_create(&cfg, &enc);
  printf("create=%d msg=%s\n", rc, rc == IE_OK ? "" : ie_last_error());
  if (rc == IE_OK) {            /* a GPU is present: the handle must be usable and destroyable */
    printf("handle max_batch=%d\n", (int)ie_encoder_max_batch(enc));
    ie_encoder_destroy(enc);
  } else if (rc != IE_ERR_CUDA || strstr(ie_last_error(), "no CPU fallback") == NULL) {
    return 3;
  }
  rc = ie_mlp_create(2, dims, 0, &mlp);
  printf("mlp_create=%d\n", rc);
  if (rc == IE_OK) ie_mlp_destroy(mlp);
  else if (rc != IE_ERR_CUDA) return 4;
  ie_encoder_destroy(NULL);     /* NULL handles are ignored */
  ie_mlp_destroy(NULL);
  return 0;
}
