"""Stand-in for mmcv (not installed): the sAP toolkit's det / track modules import it, and the forecast script's path
calls none of it."""
