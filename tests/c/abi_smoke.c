/* Plain-C consumer of include/goslam_b200.h: proves the header is valid C99 (no C++-isms), that the
 * shared library links without torch / python, and exercises the host-only helpers (no GPU needed). */
#include <stdio.h>
#include <string.h>
#include "goslam_b200.h"

int main(void) {
  int64_t offsets[17];
  int res[16];
  float scales[16];
  int fails = 0;
  if (goslam_version() <= 0) { printf("version\n"); ++fails; }
  if (goslam_sm_arch() != 90) { printf("arch %d\n", goslam_sm_arch()); ++fails; }
  if (strcmp(goslam_strerror(GOSLAM_OK), "ok") != 0) { printf("strerror\n"); ++fails; }
  if (goslam_strerror(GOSLAM_EWORKSPACE) == NULL) ++fails;
  /* workspace helpers are pure host functions */
  if (goslam_ba_workspace_bytes(36, 11, 40, 80, 1, 8) == 0) { printf("ba ws\n"); ++fails; }
  if (goslam_ba_workspace_bytes(36, 0, 40, 80, 1, 8) != 0) { printf("ba ws invalid\n"); ++fails; }
  if (goslam_ba_system_doubles(1, 8) != 42u * 42u + 42u) { printf("system doubles\n"); ++fails; }
  if (goslam_corr_level_plane_elems(0, GOSLAM_LAYOUT_TILED, 30, 40) != 8u * 10u * 16u) { printf("plane\n"); ++fails; }
  if (goslam_corr_level_plane_elems(3, GOSLAM_LAYOUT_ROWMAJOR, 40, 80) != 5u * 10u) { printf("plane rm\n"); ++fails; }
  if (goslam_proximity_workspace_bytes(0, 0, 12) == 0) { printf("prox ws\n"); ++fails; }
  if (goslam_neus_workspace_bytes(1024, 72) == 0) { printf("neus ws\n"); ++fails; }
  if (goslam_hashgrid_layout(offsets, res, scales) != 12599920) { printf("hashgrid\n"); ++fails; }
  if (res[0] != 16 || offsets[0] != 0) { printf("hashgrid level 0\n"); ++fails; }
  /* argument validation happens before any CUDA call */
  if (goslam_corr_index_forward(NULL, GOSLAM_F16, NULL, NULL, -1, 1, 1, 1, 1, 3, NULL) != GOSLAM_EINVAL) { printf("einval\n"); ++fails; }
  if (goslam_corr_index_backward() != GOSLAM_EUNSUPPORTED) { printf("unsupported\n"); ++fails; }
  if (goslam_corr_build(NULL, NULL, GOSLAM_F16, NULL, 4, 1, 128, 4, 80, NULL) != GOSLAM_EINVAL) { printf("corr_build einval\n"); ++fails; }
  if (goslam_corr_pool_build(NULL, 8, 1, NULL, NULL, NULL, NULL, 4, 1, 128, 40, 160, NULL) != GOSLAM_EINVAL) { printf("pool_build einval\n"); ++fails; }
  printf(fails ? "FAILED %d\n" : "abi smoke ok\n", fails);
  return fails;
}
