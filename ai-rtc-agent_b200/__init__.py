"""H100-native per-frame img2img path behind the lib/pipeline.py / lib/wrapper.py call surface of
yondonfu/ai-rtc-agent.  Layout:

  csrc/   hand-written sm_100a CUDA (tcgen05 / TMA / TMEM) + the C ABI (include/b200sd.h)
  host/   Python mirror of the reference's StreamDiffusionPipeline / StreamDiffusionWrapper,
          bound to libb200sd.so with ctypes

Import as `ai_rtc_agent_b200` (alias module at the repo root)."""

__version__ = "0.1.0"
