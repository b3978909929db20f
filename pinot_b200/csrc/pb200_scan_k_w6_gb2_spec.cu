// one instantiation of the scan kernel per translation unit (parallel build)
#define PB200_INST 6, true, false, 2, true
#define PB200_INST_NAME launch_scan_w6_gb2_spec
#define PB200_INST_W 6
#include "pb200_scan_inst.inc"
