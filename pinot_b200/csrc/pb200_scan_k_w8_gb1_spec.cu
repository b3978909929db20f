// one instantiation of the scan kernel per translation unit (parallel build)
#define PB200_INST 8, true, false, 1, true
#define PB200_INST_NAME launch_scan_w8_gb1_spec
#define PB200_INST_W 8
#include "pb200_scan_inst.inc"
