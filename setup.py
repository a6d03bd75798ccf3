"""Install torchacc_b200 (the native library is built in-tree by ``python -m torchacc_b200.build_native``)."""
from setuptools import find_packages, setup
from setuptools.command.build_py import build_py


class BuildWithNative(build_py):
    def run(self):
        try:
            from torchacc_b200 import build_native
            build_native.build()
        except Exception as e:  # the Python tier works without the library (CPU plumbing tests)
            print(f"[torchacc_b200] native build skipped: {e}")
        super().run()


setup(
    name="torchacc_b200",
    version="0.1.0",
    description="H100-native (sm_90a) training acceleration framework with TorchAcc's capabilities",
    packages=find_packages(include=["torchacc_b200", "torchacc_b200.*"]),
    package_data={"torchacc_b200": ["_C.so"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.5", "numpy"],
    cmdclass={"build_py": BuildWithNative},
    entry_points={"console_scripts": [
        "consolidate_and_reshard_fsdp_ckpts=torchacc_b200.utils.consolidate_and_reshard_ckpts:main",
    ]},
)
