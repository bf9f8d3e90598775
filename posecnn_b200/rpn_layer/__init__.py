# mirrors lib/rpn_layer/ of the reference (the test-time path: anchors and proposals)
