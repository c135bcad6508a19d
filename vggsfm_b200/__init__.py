"""vggsfm_b200 -- H100-native (sm_90a) geometry hot path for VGGSfM (see DESIGN.md)."""
