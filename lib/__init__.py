"""Import-compatibility package: `from lib.pipeline import StreamDiffusionPipeline` and
`from lib.wrapper import StreamDiffusionWrapper` (agent.py:23, lib/pipeline.py:9 of the reference) resolve to
the H100 implementation, so the reference's agent.py / lib/tracks.py run against it unmodified."""
