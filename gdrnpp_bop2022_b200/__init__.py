"""H100-native GDRNPP per-ROI pose inference hot path."""
