"""Import shim: `from models.emage_audio import ...` (what the reference's test_emage_audio.py:13 and
train_emage_audio.py:29 do) resolves to the H100 implementation in pantomatrix_b200."""
