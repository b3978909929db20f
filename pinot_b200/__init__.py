"""pinot_b200 -- H100-native (sm_90a) scan -> filter -> group-by-aggregate path for Apache Pinot segments (see DESIGN.md)."""
