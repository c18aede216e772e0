"""Import-time stand-in for pycocotools (not a dependency of this package): the reference's caption script imports
`pycocotools.coco.COCO` at module level (downstream/run_caption_distributed_gpt3.py:39) but only uses it to score
generated captions (CIDEr / BLEU, :283-300) - metric tooling, outside the hot path.  Training and generation run;
scoring asks for the real package.  compat/ sits at the END of sys.path, so an installed pycocotools always wins."""
