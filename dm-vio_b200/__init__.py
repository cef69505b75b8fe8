"""H100-native DM-VIO photometric hot path (package root; see DESIGN.md)."""
