"""H100 drop-in for the reference's codes/DSN modules (`model.py`, `loss.py`) and its training iteration."""
