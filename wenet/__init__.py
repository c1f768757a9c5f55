"""Drop-in import name: `import wenet; wenet.load_model(...)` resolves to the H100 engine.

The reference installs its package as `wenet` (pyproject.toml:25-32); code written against it
(`wenet.load_model`, `wenet.ReverbASR`, `wenet.get_available_models`, `wenet.download_model`,
`wenet.bin.recognize_wav:main`, `wenet.cli.reverb`) keeps working when this repository is on
sys.path instead.
"""
from reverb_b200 import ReverbASR, download_model, get_available_models, load_model  # noqa: F401
