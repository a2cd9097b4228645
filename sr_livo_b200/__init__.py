"""sr_livo_b200 — H100-native (sm_90a) LIO scan-matching hot path of SR-LIVO (see DESIGN.md)."""
