// The example handlers' entry points: compiled to an sm_90a cubin (beta9_b200.build.compile_handlers; build() makes
// beta9_b200/example_handlers.cubin) and loaded with b9_handler_load(ctx, image, size, "<name>", &id).
#include "handlers.cuh"

B9_HANDLER(echo_str, b9_examples::EchoStr)
B9_HANDLER(crc32_str, b9_examples::Crc32Str)
B9_HANDLER(word_count, b9_examples::WordCount)
B9_HANDLER(prod, b9_examples::Prod)
B9_HANDLER(greet, b9_examples::Greet)
B9_HANDLER(join, b9_examples::Join)
B9_HANDLER(field_sum, b9_examples::FieldSum)
B9_HANDLER(tokens, b9_examples::Tokens)
B9_HANDLER(grid, b9_examples::Grid)
B9_HANDLER(describe, b9_examples::Describe)
B9_HANDLER(pick, b9_examples::Pick)
