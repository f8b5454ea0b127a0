"""reagent_b200 -- H100-native (sm_90a) implementation of ReAgent's off-policy training
hot path: replay sampling -> dense preprocessing -> TD update (DQN / QR-DQN / SAC / TD3)
-> Adam + soft target update, behind ReAgent's own Python surface.  See DESIGN.md."""
__version__ = "0.1.0"
