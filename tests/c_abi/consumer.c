/* A plain-C99 consumer of include/f5_b200.h: proves the boundary is a C ABI (no C++ / torch types in the
 * signatures) that any host language can bind.  Built and run by tests/test_abi.py with gcc; without a GPU every
 * compute entry must answer F5_ERR_NO_DEVICE. */
#include <stdio.h>
#include <string.h>

#include "f5_b200.h"

int main(void) {
  int32_t sizes[10];
  int n = f5_struct_sizes(sizes, 10);
  printf("abi=%d structs=%d sizeof(f5_gemm_args)=%d/%d\n", f5_abi_version(), n, (int)sizeof(f5_gemm_args), (int)sizes[0]);
  if (n != 10 || (int)sizeof(f5_gemm_args) != sizes[0]) return 1;   /* the C compiler's layout == the library's */
  int rc = f5_device_check();
  printf("device_check=%d (%s)\n", rc, rc ? f5_last_error() : "sm_90 device present");
  f5_gemm_args g;
  memset(&g, 0, sizeof g);
  int rg = f5_gemm_bf16(&g, NULL);      /* no device: F5_ERR_NO_DEVICE; with a device: rejected as invalid (null operands) */
  printf("gemm_rc=%d (%s)\n", rg, f5_last_error());
  return rg < 0 ? 0 : 2;
}
