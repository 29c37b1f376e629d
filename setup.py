from setuptools import find_packages, setup

setup(
    name="fms_fsdp_b200",
    version="0.1.0",
    description="H100-native FSDP pre-training engine with the capabilities of foundation-model-stack/fms-fsdp",
    packages=find_packages(include=["fms_fsdp_b200*", "fms_fsdp*", "speculator*"]),
    package_data={"fms_fsdp_b200": ["csrc/*", "_C.so"]},
    py_modules=["main_training_llama", "main_training_mamba", "fms_to_hf_llama", "fms_to_hf_mamba", "hf_to_fms_llama"],
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "pyarrow", "transformers", "safetensors"],
)
