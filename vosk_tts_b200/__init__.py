"""H100-native VITS2 inference engine behind the vosk_tts Model/Synth API (hot path only)."""
