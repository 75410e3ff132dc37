"""Inference from raw recordings: ``beautify.SVBBeautifier`` runs the SVB task's a2p chain from WAV pairs to audio."""
