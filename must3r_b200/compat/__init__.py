"""Operator seams of the reference served by libm3r_b200.so (SURVEY.md §8b, INTEGRATION.md §3-4).

``must3r_b200.compat.curope``     drop-in for the reference's optional native ``curope`` module
                                  (dust3r/croco/models/curope/curope.cpp:49-69, curope2d.py:32-39).
``must3r_b200.compat.attention``  ``toggle_memory_efficient_attention`` / ``has_xformers`` of
                                  must3r/model/blocks/attention.py:5-27 and an ``attention()`` with the signature of
                                  ``CoreAttention.attention`` (:37) running on the wgmma kernel.
"""
