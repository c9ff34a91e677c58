"""abyss_b200: H100-native (sm_90a) Bloom-filter de Bruijn graph unitig stage (abyss-bloom-dbg path)."""
__version__ = "0.1.0"
