"""bflc_demo_b200 -- an H100-native (Hopper) committee-consensus federated-learning engine.

Capability parity target: iammcy/BFLC-demo (FISCO-BCOS precompiled contract + TF1 client);
see SURVEY.md for the component map and DESIGN.md for the H100 (sm_90a) architecture.
"""
__version__ = "0.1.0"
