"""fastani_b200 -- H100-native ANI hot path (reference index build + query mapping).

The product is the CUDA library fastani_b200/lib/libfastani_b200.so behind the C ABI of
include/fastani_b200.h; this package is its Python host side.  There is no CPU fallback:
importing works anywhere, but every compute call raises if the library or a GPU is missing.
"""
from .api import (Parameters, Context, Genome, PackedBatch, Sketch, Map, MapCounters, BaniError,  # noqa: F401
                  MAPPING_DTYPE, MINIMIZER_DTYPE, CGI_DTYPE, FRAG_DTYPE, compute_cgi, compute_cgi_sketched, QuerySketch,
                  load_library, library_path, compute_cgi_chunked, plan_chunks, index_footprint, index_budget,
                  map_working_set, parse_byte_count, plan_run, run_working_set, index_file_info, index_file_extend,
                  compute_cgi_from_index_file)
from .fasta import read_fasta  # noqa: F401
