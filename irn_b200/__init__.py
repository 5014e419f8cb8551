"""irn_b200: H100-native pseudo-label hot path of jiwoon-ahn/irn (see DESIGN.md)."""
__version__ = "0.1.0"
