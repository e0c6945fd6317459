/* Plain-C consumer of the text-classifier part of include/issue_emb_b200.h: the declarations are valid C, every
 * ie_clas_* entry point links from libissue_emb_b200.so, the host-only window rule answers without a GPU, and bad
 * arguments come back as error codes.  Built and run by tests/test_text_classifier_reference.py. */
#include <stdio.h>

#include "issue_emb_b200.h"

int main(void) {
  typedef void (*fn)(void);
  fn syms[] = {(fn)ie_clas_window, (fn)ie_clas_create, (fn)ie_clas_destroy, (fn)ie_clas_load_stage,
               (fn)ie_clas_forward, (fn)ie_clas_pool, (fn)ie_clas_check_errors, (fn)ie_clas_launch_count};
  int32_t dims[3] = {2400, 50, 3};
  int32_t start = -1;
  ie_clas* c = NULL;
  int rc;
  printf("clas_symbols=%d activations=%d,%d\n", (int)(sizeof syms / sizeof syms[0]), IE_CLAS_SIGMOID, IE_CLAS_SOFTMAX);
  if (ie_clas_window(1470, 70, 1400, &start) != IE_OK || start != 140) return 2;
  if (ie_clas_window(70, 70, 70, &start) != IE_ERR_INVALID) return 3;
  printf("window(1470)=140 window(70, max_len 70)=%s\n", ie_last_error());
  rc = ie_clas_create(NULL, 2, dims, IE_CLAS_SIGMOID, &c);
  if (rc != IE_ERR_INVALID || c != NULL) return 4;
  if (ie_clas_forward(NULL, NULL, NULL, NULL, 1, 1, NULL, NULL, 0, NULL) != IE_ERR_INVALID) return 5;
  if (ie_clas_launch_count(NULL) != -1) return 6;
  ie_clas_destroy(NULL); /* NULL handles are ignored */
  return 0;
}
