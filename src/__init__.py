"""Drop-in `src.*` import paths of facebookresearch/jepa, re-exported from the H100-native jepa_b200 package."""
