"""``python -m cleandiffuser_b200.run <script.py> [args...]`` -- run an unmodified reference script on the H100 engine
(installs the overlay of ``cleandiffuser_b200.overlay`` first)."""
from .overlay import main

if __name__ == "__main__":
    main()
