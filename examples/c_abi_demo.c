/* Plain-C client of the boundary (include/yolact_b200.h): what a cgo / JNI / FFI binding would do.
 *   gcc -std=c99 -Wall -Iinclude examples/c_abi_demo.c -o c_abi_demo yolact_b200/libyolact_b200.so -Wl,-rpath,$PWD/yolact_b200
 * Creates an ops-only handle (no backbone) and runs row-wise softmax on the device through the library's own
 * kernels; on a machine without an H100 it reports the library's error message and exits 0. */
#include <stdio.h>
#include <string.h>

#include "yolact_b200.h"

int main(void) {
  yb_config cfg;
  yb_handle* h = NULL;
  int rc;
  memset(&cfg, 0, sizeof(cfg));
  cfg.backbone = YB_BACKBONE_NONE;
  cfg.num_classes = 81;
  cfg.mask_dim = 32;
  cfg.precision = YB_PREC_F32;
  cfg.nms_top_k = 200;
  cfg.nms_conf_thresh = 0.05f;
  cfg.nms_thresh = 0.5f;
  cfg.max_num_detections = 100;
  cfg.max_size = 550;
  rc = yb_device_count(); /* >= 0: devices, < 0: a yb_status */
  printf("yolact_b200 ABI %d, %d CUDA device(s)\n", yb_abi_version(), rc < 0 ? 0 : rc);
  rc = yb_create(&cfg, 0, &h);
  if (rc != YB_OK) {
    printf("yb_create: status %d (%s)\n", rc, yb_last_error());
    return 0; /* no device here: the product has no CPU fallback, by design */
  }
  printf("handle created, %lld kernel launches so far\n", (long long)yb_launch_count(h));
  yb_destroy(h);
  return 0;
}
