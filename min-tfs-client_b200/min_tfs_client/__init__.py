"""H100-native drop-in for zendesk/min-tfs-client's Predict hot path (same import name)."""
