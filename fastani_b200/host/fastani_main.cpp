// fastani_main.cpp -- the fastANI command line on top of libfastani_b200.so.
//
// Same options and output files as the reference CLI (src/map/include/parseCmdArgs.hpp:118-256,
// src/cgi/core_genome_identity.cpp:27-167): -q/--query, --ql/--queryList, -r/--ref, --rl/--refList, -o/--output,
// -k/--kmer, --fragLen, --minFraction, --maxRatioDiff, --visualize, --matrix, -t/--threads, -s/--sanityCheck,
// -v/--version, -h/--help.  Differences, all on the host side:
//   * the reference list is split over GPUs (--gpus N, default: every visible device), not over OpenMP threads;
//     -t sets the host threads of the ingest stage.  Results do not depend on the split (SURVEY.md section 0-3).
//   * every genome file is read ONCE (parallel inflate + parse), its length for the --minFraction filter comes from
//     the same pass (the reference reads each file again in computeGenomeLengths, computeCoreIdentity.hpp:48-92)
//   * --saveIndex / --loadIndex: the on-disk sketch cache the reference lacks (its only answer to repeated runs is
//     scripts/splitDatabase.sh + README.md:104-106); parameters (k, fragLen, window) are stored and a mismatch is refused
//   * the per-pair reduction runs on the device for every query of a GPU at once (bani_map_cgi_sketch); with --visualize
//     it also returns the 2-way fragment mappings the .visual file is written from (bani_map_cgi_sketch_frags).
//     BANI_CLI_HOST_CGI=1 (a test switch) instead maps one query at a time, copies its mapping rows back and runs
//     cgi::computeCGI on the host, so that both paths can be compared on the same inputs.  The same switch makes a
//     --loadIndex run read and hash every query file, also those of genomes of the index (whose sketches are otherwise
//     derived from the shard file that holds them)
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <sstream>
#include <thread>
#include <unistd.h>
#include "ani_host.hpp"

using namespace skch;
typedef std::chrono::high_resolution_clock Clock;

static void usage(const char *prog, std::ostream &o)
{
  o << "-----------------\n"
       "fastANI (H100-native engine): alignment-free whole-genome Average Nucleotide Identity (ANI)\n"
       "-----------------\n"
       "Example usage:\n"
       "$ " << prog << " -q genome1.fa -r genome2.fa -o output.txt\n"
       "$ " << prog << " -q genome1.fa --rl genome_list.txt -o output.txt\n\n"
       "OPTIONS\n"
       "     -h, --help            print this help page\n"
       "     -r, --ref <value>     reference genome (fasta/fastq)[.gz]\n"
       "     --rl, --refList <value>   a file containing list of reference genome files, one genome per line\n"
       "     -q, --query <value>   query genome (fasta/fastq)[.gz]\n"
       "     --ql, --queryList <value> a file containing list of query genome files, one genome per line\n"
       "     -k, --kmer <value>    kmer size <= 32 [default : 16]\n"
       "     -t, --threads <value> host threads for reading the genome files [default : 1]\n"
       "     --gpus <value>        GPUs to split the reference list over [default : all visible]\n"
       "     --fragLen <value>     fragment length [default : 3,000]\n"
       "     --minFraction <value> minimum fraction of genome that must be shared for trusting ANI [default : 0.2]\n"
       "     --maxRatioDiff <value> maximum difference between (Total Ref. Length/Total Occ. Hashes) and\n"
       "                           (Total Ref. Length/Total No. Hashes) [default : 100.0]\n"
       "     --partition <value>   how the reference list is cut into one shard per GPU: interleave (the reference's round-robin\n"
       "                           deal, default) or block (contiguous ranges: list neighbours stay on one GPU)\n"
       "     --saveIndex <prefix>  write the reference sketches to <prefix>.meta + <prefix>.<shard>of<N>.idx after building them\n"
       "     --loadIndex <prefix>  take the references from a saved index instead of -r/--rl: no reference file is read or\n"
       "                           sketched again; queries that are genomes of the index need no file either.\n"
       "                           Shard files are loaded in chunks that fit the device, on as many GPUs as are visible\n"
       "     --loadIndex <old> -r/--rl <new genomes> --saveIndex <new>\n"
       "                           add genomes to a saved index: <new> holds <old>'s genomes, then the new ones, as a fresh\n"
       "                           --saveIndex of the whole list would (same shards and partition); only the new genomes are\n"
       "                           read and sketched.  The run then maps the queries against <new>\n"
       "     --visualize           output mappings for visualization (<output>.visual)\n"
       "     --matrix              also output ANI values as lower triangular matrix (<output>.matrix)\n"
       "     -o, --output <value>  output file name\n"
       "     -s, --sanityCheck     run sanity check\n"
       "     -v, --version         show version\n";
}

static std::string trim(const std::string &s)
{
  size_t a = 0, b = s.size();
  while (a < b && isspace((unsigned char)s[a])) a++;
  while (b > a && isspace((unsigned char)s[b - 1])) b--;
  return s.substr(a, b - a);
}

static void parseFileList(const std::string &fileToRead, std::vector<std::string> &fileList)   // parseCmdArgs.hpp:34-52
{
  std::ifstream in(fileToRead);
  if (in.fail()) { std::cerr << "ERROR, skch::parseFileList, Could not open " << fileToRead << "\n"; exit(1); }
  std::string line;
  while (std::getline(in, line)) { line = trim(line); if (!line.empty()) fileList.push_back(line); }
}

static void validateInputFiles(const std::vector<std::string> &q, const std::vector<std::string> &r)   // parseCmdArgs.hpp:59-90
{
  if (q.empty() || r.empty()) { std::cerr << "ERROR, skch::validateInputFiles, Count of query and ref genomes should be non-zero" << std::endl; exit(1); }
  for (const auto *lst : {&q, &r})
    for (const auto &e : *lst) { std::ifstream in(e); if (in.fail()) { std::cerr << "ERROR, skch::validateInputFiles, Could not open " << e << std::endl; exit(1); } }
}

static void parseandSave(int argc, char **argv, Parameters &p)
{
  std::string refName, refList, qryName, qryList;
  bool help = false, version = false;
  auto need = [&](int &i) -> const char * { if (i + 1 >= argc) { usage(argv[0], std::cout); exit(1); } return argv[++i]; };
  for (int i = 1; i < argc; i++) {
    const std::string a = argv[i];
    if (a == "-h" || a == "--help") help = true;
    else if (a == "-r" || a == "--ref") refName = need(i);
    else if (a == "--rl" || a == "--refList") refList = need(i);
    else if (a == "-q" || a == "--query") qryName = need(i);
    else if (a == "--ql" || a == "--queryList") qryList = need(i);
    else if (a == "-k" || a == "--kmer") p.kmerSize = atoi(need(i));
    else if (a == "-t" || a == "--threads") p.threads = atoi(need(i));
    else if (a == "--gpus") p.gpus = atoi(need(i));
    else if (a == "--fragLen") p.minReadLength = atoi(need(i));
    else if (a == "--minFraction") p.minFraction = (float)atof(need(i));
    else if (a == "--maxRatioDiff") p.maxRatioDiff = (float)atof(need(i));
    else if (a == "--partition") { const std::string v = need(i); if (v == "block") p.blockPartition = true; else if (v != "interleave") { usage(argv[0], std::cout); exit(1); } }
    else if (a == "--saveIndex") p.saveIndex = need(i);
    else if (a == "--loadIndex") p.loadIndex = need(i);
    else if (a == "--visualize") p.visualize = true;
    else if (a == "--matrix") p.matrixOutput = true;
    else if (a == "-o" || a == "--output") p.outFileName = need(i);
    else if (a == "-s" || a == "--sanityCheck") p.sanityCheck = true;
    else if (a == "-v" || a == "--version") version = true;
    else { usage(argv[0], std::cout); exit(1); }
  }
  if (help) { usage(argv[0], std::cout); exit(0); }
  if (version) { std::cerr << "version 1.33 (" << bani_version() << ")\n\n"; exit(0); }
  const bool refsGiven = !refName.empty() || !refList.empty();
  if (!p.loadIndex.empty() && refsGiven && p.saveIndex.empty()) { std::cerr << "ERROR, --loadIndex replaces -r/--rl: give one of them\n"; exit(1); }
  if (!p.loadIndex.empty() && !p.saveIndex.empty() && !refsGiven) { std::cerr << "ERROR, --saveIndex and --loadIndex exclude each other\n"; exit(1); }
  if (!p.loadIndex.empty() && p.saveIndex == p.loadIndex) {
    std::cerr << "ERROR, --saveIndex " << p.saveIndex << " is the index given to --loadIndex: the index with the added genomes goes to a new prefix\n";
    exit(1);
  }
  if (refName.empty() && refList.empty() && p.loadIndex.empty()) { std::cerr << "Provide reference file (s)\n"; exit(1); }
  if (qryName.empty() && qryList.empty()) { std::cerr << "Provide query file (s)\n"; exit(1); }
  if (!refName.empty()) p.refSequences.push_back(refName); else if (!refList.empty()) parseFileList(refList, p.refSequences);
  if (!qryName.empty()) p.querySequences.push_back(qryName); else parseFileList(qryList, p.querySequences);
  if (!(p.minFraction >= 0.0f && p.minFraction <= 1.0f)) { std::cerr << "ERROR, --minFraction must lie in [0, 1]\n"; exit(1); }
  if (p.threads < 1) p.threads = 1;
  bani_params c = p.c();
  const int w = bani_recommended_window_size(&c);          // Stat::recommendedWindowSize, parseCmdArgs.hpp:244-247
  if (w < 0) { std::cerr << "ERROR, " << bani_last_error() << "\n"; exit(1); }
  p.windowSize = w;
  std::cerr << ">>>>>>>>>>>>>>>>>>\nReference = [" ;
  for (size_t i = 0; i < p.refSequences.size(); i++) std::cerr << (i ? ", " : "") << p.refSequences[i];
  std::cerr << "]\nQuery = [";
  for (size_t i = 0; i < p.querySequences.size(); i++) std::cerr << (i ? ", " : "") << p.querySequences[i];
  std::cerr << "]\nKmer size = " << p.kmerSize << "\nFragment length = " << p.minReadLength << "\nThreads = " << p.threads
            << "\nANI output file = " << p.outFileName << "\nSanity Check  = " << p.sanityCheck << "\n>>>>>>>>>>>>>>>>>>" << std::endl;
  if (p.loadIndex.empty()) validateInputFiles(p.querySequences, p.refSequences);
  else for (const auto &e : p.refSequences) {       // genomes added to a loaded index (queries may be genomes of the index)
    std::ifstream in(e);
    if (in.fail()) { std::cerr << "ERROR, skch::validateInputFiles, Could not open " << e << std::endl; exit(1); }
  }
}

// ---- metadata of a saved index: what the flat per-shard files (bani_index_save) do not hold -- genome paths and
//      contig names -- plus the parameters, so that a mismatch is reported before any GPU work
struct IndexMeta {
  int k = 0, fragLen = 0, window = 0, shards = 0;
  bool block = false;                                                 // version 2: the shards are contiguous blocks of the list
  std::vector<std::string> refPaths;                                  // global reference order
  std::vector<std::vector<std::string>> contigNames;                  // per shard, seqId order
};
static std::string shardFile(const std::string &prefix, int g, int G) { return prefix + "." + std::to_string(g) + "of" + std::to_string(G) + ".idx"; }

static void writeMeta(const std::string &prefix, const Parameters &p, int G, const std::vector<std::vector<std::string>> &contigNames)
{
  std::ofstream o(prefix + ".meta");
  if (!o) throw std::runtime_error("cannot write " + prefix + ".meta");
  o << "BANI_INDEX_META\t" << (p.blockPartition ? 2 : 1) << "\n" << p.kmerSize << "\t" << p.minReadLength << "\t" << p.windowSize << "\t" << G << "\t" << p.refSequences.size() << "\n";
  for (const auto &r : p.refSequences) o << r << "\n";
  for (int g = 0; g < G; g++) { o << contigNames[g].size() << "\n"; for (const auto &n : contigNames[g]) o << n << "\n"; }
}

static IndexMeta readMeta(const std::string &prefix)
{
  std::ifstream in(prefix + ".meta");
  if (!in) throw std::runtime_error("cannot open " + prefix + ".meta");
  IndexMeta m; std::string tag; int ver = 0; size_t nRefs = 0;
  in >> tag >> ver >> m.k >> m.fragLen >> m.window >> m.shards >> nRefs;
  if (!in || tag != "BANI_INDEX_META" || (ver != 1 && ver != 2) || m.shards < 1) throw std::runtime_error(prefix + ".meta is not an index metadata file");
  m.block = ver == 2;
  std::string line; std::getline(in, line);
  for (size_t i = 0; i < nRefs; i++) { if (!std::getline(in, line)) throw std::runtime_error(prefix + ".meta is truncated"); m.refPaths.push_back(line); }
  m.contigNames.resize(m.shards);
  for (int g = 0; g < m.shards; g++) {
    if (!std::getline(in, line)) throw std::runtime_error(prefix + ".meta is truncated");
    const size_t n = (size_t)std::stoull(line);
    for (size_t i = 0; i < n; i++) { if (!std::getline(in, line)) throw std::runtime_error(prefix + ".meta is truncated"); m.contigNames[g].push_back(line); }
  }
  return m;
}

int main(int argc, char **argv)
{
  if (argc == 3 && std::string(argv[1]) == "--dumpContigs") {       // test hook for the reader: name, length, crc32 per contig
    try {
      const bani_host::HostGenome g = bani_host::read_genome(argv[2]);
      for (const auto &c : g.contigs)
        std::cout << c.name << "\t" << c.len << "\t" << crc32(0L, g.seq.data() + c.off, (uInt)c.len) << "\n";
      return 0;
    } catch (const std::exception &e) { std::cerr << "ERROR, " << e.what() << std::endl; return 1; }
  }
  if (argc == 3 && std::string(argv[1]) == "--selftestWriters") {   // test hook for the writers (no GPU needed): a fixed result set
    Parameters p;
    p.querySequences = {"q/a.fa", "q/b.fa", "r/c.fa"}; p.refSequences = {"r/c.fa", "q/a.fa", "r/d.fa"};
    p.minReadLength = 3000; p.minFraction = 0.2f; p.matrixOutput = true;
    std::unordered_map<std::string, uint64_t> len = {{"q/a.fa", 150000}, {"q/b.fa", 90000}, {"r/c.fa", 150000}, {"r/d.fa", 3000000}};
    std::vector<cgi::CGI_Results> v = {
      {0, 0, 40, 50, 97.75071f}, {1, 0, 50, 50, 100.0f}, {2, 0, 9, 50, 81.5f},          // a -> c, a -> a (self), a -> d (fails minFraction: 27000 < 30000)
      {0, 1, 20, 30, 88.123456f}, {2, 1, 6, 30, 80.0f},                                  // b -> c, b -> d (18000 >= 18000 passes)
      {1, 2, 45, 50, 97.5f}, {0, 2, 50, 50, 100.0f}};                                    // c -> a (averaged with a -> c in the matrix), c -> c (self)
    cgi::outputCGI(p, len, v, argv[2]);
    cgi::outputPhylip(p, len, v, argv[2]);
    return 0;
  }
  const auto tStart = Clock::now();
  Parameters parameters;
  parseandSave(argc, argv, parameters);
  const std::string fileName = parameters.outFileName;
  try {
    const bool loading = !parameters.loadIndex.empty();
    const bool extending = loading && !parameters.saveIndex.empty();      // -r/--rl genomes added to the loaded index
    IndexMeta meta;
    std::vector<std::string> addedRefs;
    if (loading) {
      meta = readMeta(parameters.loadIndex);
      if (meta.k != parameters.kmerSize || meta.fragLen != parameters.minReadLength || meta.window != parameters.windowSize)
        throw std::runtime_error("the saved index was built with k " + std::to_string(meta.k) + " fragLen " + std::to_string(meta.fragLen) + " window " + std::to_string(meta.window) +
                                 ", this run asks for k " + std::to_string(parameters.kmerSize) + " fragLen " + std::to_string(parameters.minReadLength) + " window " + std::to_string(parameters.windowSize));
      if (extending && meta.block && meta.shards > 1)
        throw std::runtime_error("cannot add genomes to " + parameters.loadIndex + ": its " + std::to_string(meta.shards) + " shards are blocks of the reference "
                                 "list (--partition block), and a fresh save of the longer list would cut the blocks differently");
      addedRefs = parameters.refSequences;
      parameters.refSequences = meta.refPaths;
      parameters.refSequences.insert(parameters.refSequences.end(), addedRefs.begin(), addedRefs.end());
      parameters.blockPartition = meta.block;
    }
    // a run that names its GPU count initialises only those devices (the driver's start-up cost grows with every visible GPU)
    {
      const int want = loading ? (parameters.gpus > 0 ? std::min(parameters.gpus, meta.shards) : meta.shards) : parameters.gpus;
      if (want > 0 && !getenv("CUDA_VISIBLE_DEVICES")) {
        std::string v; for (int g = 0; g < want; g++) v += (g ? "," : "") + std::to_string(g);
        setenv("CUDA_VISIBLE_DEVICES", v.c_str(), 0);
      }
    }
    int32_t nDev = 0;
    if (bani_device_count(&nDev) != BANI_OK || nDev == 0) throw std::runtime_error("no CUDA device available (this program has no CPU path)");
    // S reference shards: one per GPU, or the saved index's shard files, of which GPU g takes g, g + G, ... in turn
    const int visible = parameters.gpus > 0 ? std::min(parameters.gpus, (int)nDev) : (int)nDev;
    const int G = loading ? std::min(visible, meta.shards) : visible;
    const int S = loading ? meta.shards : G;
    const auto shards = cgi::splitReferenceGenomes((int)parameters.refSequences.size(), S, parameters.blockPartition);
    // the contexts (CUDA context creation, stream set-up) come up while the reader threads parse and pack the files
    std::vector<bani_ctx *> ctxs(G, nullptr); std::vector<std::string> ctxErr(G);
    std::vector<std::thread> ctxThreads;
    for (int g = 0; g < G; g++)
      ctxThreads.emplace_back([&, g]() { bani_params cp = parameters.c(); if (bani_ctx_create(g, &cp, &ctxs[g]) != BANI_OK) ctxErr[g] = bani_last_error(); });

    // ---- ingest: every distinct file once, in parallel.  With a loaded index no reference file is read, and neither is
    //      a member query -- one whose path is a genome of the index (its first position in the list): its sketch is derived
    //      from the shard file that holds the genome
    auto t0 = Clock::now();
    std::unordered_map<std::string, int> refOrdinal;                  // path -> first position in the reference list
    for (size_t j = 0; j < parameters.refSequences.size(); j++) refOrdinal.emplace(parameters.refSequences[j], (int)j);
    const char *hostCgiEnv = getenv("BANI_CLI_HOST_CGI");
    const bool hostCgiSwitch = hostCgiEnv && atoi(hostCgiEnv) != 0;
    const bool hostCgi = parameters.visualize && hostCgiSwitch;         // per-query host computeCGI (test switch)
    const bool deriveQueries = loading && !hostCgiSwitch;
    std::vector<std::pair<int, int>> memberAt(parameters.querySequences.size(), {-1, -1});     // (shard file, ordinal) of a member query
    if (deriveQueries)
      for (size_t q = 0; q < memberAt.size(); q++) {
        const auto it = refOrdinal.find(parameters.querySequences[q]);
        if (it != refOrdinal.end()) memberAt[q] = cgi::referenceShardOrdinal(it->second, (int)parameters.refSequences.size(), S, parameters.blockPartition);
      }
    auto derivable = [&](size_t q) { return memberAt[q].first >= 0; };
    std::unordered_map<std::string, int> pathId; std::vector<std::string> paths;
    for (size_t q = 0; q < parameters.querySequences.size(); q++) {
      const std::string &e = parameters.querySequences[q];
      if (!derivable(q) && !pathId.count(e)) { pathId[e] = (int)paths.size(); paths.push_back(e); }
    }
    for (const auto &e : loading ? addedRefs : parameters.refSequences) if (!pathId.count(e)) { pathId[e] = (int)paths.size(); paths.push_back(e); }
    std::vector<bani_host::HostGenome> genomes(paths.size());
    {
      std::atomic<size_t> next(0); std::mutex emu; std::string err;
      auto work = [&]() {
        for (size_t i; (i = next++) < paths.size();) {
          try { genomes[i] = bani_host::read_genome(paths[i]); skch::pack_genome(genomes[i]); }     // parse + 2-bit pack in the reader thread
          catch (const std::exception &e) { std::lock_guard<std::mutex> l(emu); err = e.what(); }
        }
      };
      std::vector<std::thread> th;
      for (int i = 0; i < std::min<int>(parameters.threads, (int)paths.size()); i++) th.emplace_back(work);
      for (auto &t : th) t.join();
      for (auto &t : ctxThreads) t.join();
      if (!err.empty()) throw std::runtime_error(err);
    }
    std::unordered_map<std::string, uint64_t> genomeLengths;
    for (size_t i = 0; i < paths.size(); i++) genomeLengths[paths[i]] = cgi::genomeLength(genomes[i], parameters.minReadLength);
    std::cerr << "INFO, skch::main, Time spent reading " << paths.size() << " genome files : "
              << std::chrono::duration<double>(Clock::now() - t0).count() << " sec" << std::endl;
    for (int g = 0; g < G; g++) if (!ctxs[g]) throw std::runtime_error("bani_ctx_create: " + ctxErr[g]);

    // ---- genomes added to a saved index: shard file s of the loaded prefix, followed by the added genomes the saved partition
    //      deals to shard s (list position j goes to shard j mod S), is written to the new prefix by bani_index_file_extend --
    //      the saved genomes are not sketched again -- and .meta last.  On any failure no file of the new prefix is left.  The
    //      run then goes on as a --loadIndex run of the new prefix.
    if (extending) {
      const int nOld = (int)meta.refPaths.size();
      std::vector<char> written(S, 0);
      std::mutex xmu; std::string xerr;
      auto extendShard = [&](bani_ctx *ctx, int g, int s) {
        const std::string in = shardFile(parameters.loadIndex, s, S), out = shardFile(parameters.saveIndex, s, S);
        std::vector<const bani_host::HostGenome *> rh;
        size_t nSaved = 0;
        for (int j : shards[s]) { if (j < nOld) nSaved++; else rh.push_back(&genomes[pathId.at(parameters.refSequences[j])]); }
        const IndexFileTables t = indexFileTables(in);
        if (t.genomeLen.size() != nSaved)
          throw std::runtime_error(in + " holds " + std::to_string(t.genomeLen.size()) + " genomes, " + parameters.loadIndex + ".meta gives its shard " + std::to_string(nSaved));
        std::vector<std::unique_ptr<DeviceGenome>> dev;
        upload_genomes(ctx, rh, dev, (size_t)1 << 28, std::max(1, parameters.threads / G));
        std::vector<bani_genome *> hs; for (auto &d : dev) hs.push_back(d->h);
        const int32_t n = (int32_t)hs.size();
        auto tooMany = [&](const std::string &why) {
          return std::runtime_error("the " + std::to_string(n) + " genome(s) added to shard " + std::to_string(s) + " (" + out + ") do not fit one index: " + why +
                                    ": add fewer genomes per run");
        };
        bani_index *ix = nullptr;
        if (n == 0) check(bani_index_build(ctx, nullptr, 0, &ix), "bani_index_build");
        else {     // one index at the budget a run plans for these genomes
          std::vector<uint64_t> rlen; std::vector<int32_t> rcont;
          for (const auto *h : rh) { uint64_t len = 0; for (const auto &c : h->contigs) len += c.len; rlen.push_back(len); rcont.push_back((int32_t)h->contigs.size()); }
          std::vector<int32_t> cEnd(n); int32_t nc = 0, nb = 0; uint64_t budget = 0;
          if (bani_ctx_plan_run(ctx, 0, 0, rlen.data(), rcont.data(), n, nullptr, nullptr, 0, cEnd.data(), &nc, nullptr, &nb, &budget) != BANI_OK)
            throw tooMany(bani_last_error());
          int32_t taken = n;
          const int rc = budget ? bani_index_build_budget(ctx, hs.data(), n, budget, &ix, &taken, nullptr) : bani_index_build(ctx, hs.data(), n, &ix);
          if (rc == BANI_ERR_LIMIT) throw tooMany(bani_last_error());
          check(rc, "bani_index_build_budget");
          if (taken < n) {
            bani_index_destroy(ix);
            throw tooMany("the index budget of " + std::to_string(budget) + " bytes holds the first " + std::to_string(taken));
          }
        }
        std::unique_ptr<bani_index, void (*)(bani_index *)> ixOwner(ix, bani_index_destroy);
        uint64_t added = 0;
        check(bani_index_stats(ix, &added, nullptr, nullptr, nullptr, nullptr), "bani_index_stats");
        check(bani_index_file_extend(ctx, in.c_str(), ix, out.c_str()), "bani_index_file_extend");
        written[s] = 1;
        ixOwner.reset(); dev.clear();
        check(bani_ctx_trim(ctx), "bani_ctx_trim");
        for (const auto *h : rh) for (const auto &c : h->contigs) meta.contigNames[s].push_back(c.name);
        std::lock_guard<std::mutex> l(xmu);
        std::cerr << "INFO [GPU " << g << "], skch::main, shard file " << s << ": " << n << " genome(s) and " << added << " minimizers added to "
                  << in << " -> " << out << std::endl;
      };
      {
        std::vector<std::thread> th;
        for (int g = 0; g < G; g++)
          th.emplace_back([&, g]() {
            try { for (int s = g; s < S; s += G) extendShard(ctxs[g], g, s); }
            catch (const std::exception &e) { std::lock_guard<std::mutex> l(xmu); xerr = e.what(); }
          });
        for (auto &t : th) t.join();
      }
      auto removeWritten = [&]() { for (int s = 0; s < S; s++) if (written[s]) std::remove(shardFile(parameters.saveIndex, s, S).c_str()); };
      if (!xerr.empty()) { removeWritten(); throw std::runtime_error(xerr); }
      try { writeMeta(parameters.saveIndex, parameters, S, meta.contigNames); }
      catch (...) { removeWritten(); std::remove((parameters.saveIndex + ".meta").c_str()); throw; }
      meta.refPaths = parameters.refSequences;
      parameters.loadIndex = parameters.saveIndex;
      parameters.saveIndex.clear();
    }

    // ---- a loaded index: the tables of every shard file, read once -- the genome sizes of the run plans (a member query's
    //      from the file that holds it), the --minFraction lengths and the contig lengths of the member queries' .visual lines
    std::vector<IndexFileTables> fileTables;
    if (loading)
      for (int s = 0; s < S; s++) {
        const std::string file = shardFile(parameters.loadIndex, s, S);
        fileTables.push_back(indexFileTables(file));
        const IndexFileTables &t = fileTables.back();
        if (t.genomeLen.size() != shards[s].size())
          throw std::runtime_error(file + " holds " + std::to_string(t.genomeLen.size()) + " genomes, " + parameters.loadIndex + ".meta gives its shard " +
                                   std::to_string(shards[s].size()));
        for (size_t i = 0; i < shards[s].size(); i++) {
          const int c0 = i ? t.seqsByFile[i - 1] : 0;
          genomeLengths.emplace(parameters.refSequences[shards[s][i]], cgi::genomeLength(t.contigLen, c0, t.seqsByFile[i], parameters.minReadLength));
        }
      }

    std::vector<cgi::CGI_Results> finalResults;
    std::vector<std::string> visual(S);
    std::vector<char> sanity(S, 1); std::vector<float> ratioDiffs(S, 1.0f);
    std::vector<std::vector<std::string>> savedContigNames(S);
    std::mutex mu; std::string err;

    std::vector<std::vector<std::string>> chunkSanity(S);             // -s verdicts of chunked shards ("SPLIT s chunk c ...")

    // One chunk's index against one query block's sketches: the -s verdict (reported for the first block), and the results
    // with chunk-local reference ordinals moved to shard-local ones (+ first)
    auto mapChunk = [&](bani_ctx *ctx, int s, int chunkNo, bool firstBlock, bani_index *ix, int first, const std::vector<bani_qsketch *> &sk,
                        std::vector<cgi::CGI_Results> &local) {
      float diff = 1.0f;
      const bool sane = !parameters.sanityCheck || Sketch::indexSanityCheck(ix, parameters.maxRatioDiff, diff);
      if (!sane && firstBlock) {
        std::lock_guard<std::mutex> l(mu);
        std::ostringstream m;                                       // the stream formatting of the per-split line
        m << "ERROR :: SPLIT " << s << " chunk " << chunkNo << "'s ratio difference " << diff << " exceeds maximum thresholds.";
        chunkSanity[s].push_back(m.str());
      }
      if (!sane) return;
      bani_cgi_result *res = nullptr; uint64_t n = 0; bani_map_counters ctr;
      check(bani_map_cgi_sketch(ctx, ix, sk.data(), (int32_t)sk.size(), &res, &n, &ctr), "bani_map_cgi_sketch");
      for (uint64_t i = 0; i < n; i++)
        local.push_back(cgi::CGI_Results{first + res[i].refGenomeId, res[i].qryGenomeId, res[i].countSeq, res[i].totalQueryFragments, res[i].identity});
      bani_free(res);
    };

    // The sketch of the queries of block [q0, q1) that are read from their files (null if there are none): they are hashed
    // and their device genomes freed again
    auto hashedSketch = [&](bani_ctx *ctx, int q0, int q1, int threads) {
      std::vector<const bani_host::HostGenome *> qh; std::vector<int32_t> qid;
      for (int q = q0; q < q1; q++)
        if (!derivable(q)) { qh.push_back(&genomes[pathId.at(parameters.querySequences[q])]); qid.push_back(q); }
      bani_qsketch *qsk = nullptr;
      if (!qh.empty()) {
        std::vector<std::unique_ptr<DeviceGenome>> dq;
        upload_genomes(ctx, qh, dq, (size_t)1 << 28, threads);
        std::vector<bani_genome *> hs; for (auto &d : dq) hs.push_back(d->h);
        check(bani_qsketch_create(ctx, hs.data(), (int32_t)hs.size(), qid.data(), nullptr, &qsk), "bani_qsketch_create");
      }
      return qsk;
    };

    // The sketches of the member queries of block [q0, q1), derived from the shard files that hold them: one
    // bani_qsketch_from_index_file call per file, which reads only those genomes and checks each against its checksum.  A
    // GPU keeps the sketches of its most recent block range, so that the shard files it maps in turn with the same query
    // blocks derive them once.
    struct MemberSketches {
      int q0 = -1, q1 = -1;
      std::vector<bani_qsketch *> sk;
      void clear() { for (auto *x : sk) bani_qsketch_destroy(x); sk.clear(); q0 = q1 = -1; }
    };
    std::vector<MemberSketches> memberCache(G);
    auto memberSketches = [&](bani_ctx *ctx, int g, int q0, int q1) -> const std::vector<bani_qsketch *> & {
      MemberSketches &c = memberCache[g];
      if (c.q0 == q0 && c.q1 == q1) return c.sk;
      c.clear();
      std::vector<std::vector<int32_t>> ord(S), qid(S);
      for (int q = q0; q < q1; q++)
        if (derivable(q)) { ord[memberAt[q].first].push_back(memberAt[q].second); qid[memberAt[q].first].push_back(q); }
      for (int f = 0; f < S; f++) {
        if (ord[f].empty()) continue;
        const std::string file = shardFile(parameters.loadIndex, f, S);
        bani_qsketch *x = nullptr;
        if (bani_qsketch_from_index_file(ctx, file.c_str(), ord[f].data(), (int32_t)ord[f].size(), qid[f].data(), &x) == BANI_OK) { c.sk.push_back(x); continue; }
        std::string why = bani_last_error(), who = "one of " + std::to_string(ord[f].size()) + " query genomes";
        for (size_t i = 0; i < ord[f].size(); i++) {           // name the member whose records fail
          bani_qsketch *y = nullptr;
          if (bani_qsketch_from_index_file(ctx, file.c_str(), &ord[f][i], 1, &qid[f][i], &y) == BANI_OK) { bani_qsketch_destroy(y); continue; }
          why = bani_last_error(); who = "query genome " + parameters.querySequences[qid[f][i]];
          break;
        }
        throw std::runtime_error("cannot derive the sketch of " + who + " from " + file + ": " + why);
      }
      c.q0 = q0; c.q1 = q1;
      return c.sk;
    };

    // A shard whose index does not fit the device at once.  Per query block: the block's sketches are made; then the shard's
    // references are walked in chunks -- built from uploads (the longest prefix of the planned genomes that fits the index
    // budget: genomes it did not take stay uploaded for the next chunk) or loaded from the shard's saved file (the longest
    // run from `first` that fits) -- each mapped, and the index and the cached blocks handed back before the next chunk.
    // Results carry shard-local reference ordinals, as those of one index would.
    auto chunkedShard = [&](bani_ctx *ctx, int g, int s, const std::vector<int> &shard, const std::vector<std::pair<int, int>> &chunks,
                            const std::vector<std::pair<int, int>> &blocks, uint64_t indexBudget, std::vector<cgi::CGI_Results> &local) {
      const int threads = std::max(1, parameters.threads / G);
      const std::string file = loading ? shardFile(parameters.loadIndex, s, S) : std::string();
      int chunkNo = 0;
      for (size_t b = 0; b < blocks.size(); b++) {
        std::unique_ptr<bani_qsketch, void (*)(bani_qsketch *)> hashed(hashedSketch(ctx, blocks[b].first, blocks[b].second, threads), bani_qsketch_destroy);
        std::vector<bani_qsketch *> sk;
        if (hashed) sk.push_back(hashed.get());
        if (deriveQueries) { const auto &m = memberSketches(ctx, g, blocks[b].first, blocks[b].second); sk.insert(sk.end(), m.begin(), m.end()); }
        std::vector<std::unique_ptr<DeviceGenome>> pending;
        int first = 0;
        size_t next = 0;
        while (loading ? first < (int)shard.size() : (next < chunks.size() || !pending.empty())) {
          bani_index *ix = nullptr; int32_t taken = 0; uint64_t peak = 0;
          if (loading) check(bani_index_load_budget(ctx, file.c_str(), first, indexBudget, &ix, &taken, &peak), "bani_index_load_budget");
          else {
            if (pending.empty()) {
              std::vector<const bani_host::HostGenome *> rh;
              for (int i = chunks[next].first; i < chunks[next].second; i++) rh.push_back(&genomes[pathId.at(parameters.refSequences[shard[i]])]);
              upload_genomes(ctx, rh, pending, (size_t)1 << 28, threads);
              first = chunks[next].first;
              next++;
            }
            std::vector<bani_genome *> hs; for (auto &d : pending) hs.push_back(d->h);
            check(bani_index_build_budget(ctx, hs.data(), (int32_t)hs.size(), indexBudget, &ix, &taken, &peak), "bani_index_build_budget");
            pending.erase(pending.begin(), pending.begin() + taken);
          }
          std::unique_ptr<bani_index, void (*)(bani_index *)> ixOwner(ix, bani_index_destroy);
          mapChunk(ctx, s, chunkNo, b == 0, ix, first, sk, local);
          ixOwner.reset();
          check(bani_ctx_trim(ctx), "bani_ctx_trim");
          first += taken;
          chunkNo++;
        }
      }
    };

    // reference shard s on GPU g (g == s unless a saved index has more shard files than the run has GPUs)
    auto shardRun = [&](bani_ctx *ctx, int g, int s) {
      auto t1 = Clock::now();
      // ---- chunk plan: does the shard's index fit next to the query sketches and the mapping working set?
      std::vector<std::pair<int, int>> chunks(1, {0, (int)shards[s].size()}), blocks(1, {0, (int)parameters.querySequences.size()});
      uint64_t indexBudget = 0;
      const auto &qs = parameters.querySequences;
      std::vector<uint64_t> qlen(qs.size()), rlen; std::vector<int32_t> rcont;
      if (loading) { rlen = fileTables[s].genomeLen; rcont = fileTables[s].genomeContigs; }     // the saved shard file's genome sizes
      else {
        for (int j : shards[s]) {
          const auto &h = genomes[pathId.at(parameters.refSequences[j])];
          uint64_t len = 0; for (const auto &c : h.contigs) len += c.len;
          rlen.push_back(len); rcont.push_back((int32_t)h.contigs.size());
        }
      }
      for (size_t q = 0; q < qs.size(); q++) {
        if (derivable(q)) { qlen[q] = fileTables[memberAt[q].first].genomeLen[memberAt[q].second]; continue; }     // from the file that holds it
        for (const auto &c : genomes[pathId.at(qs[q])].contigs) qlen[q] += c.len;
      }
      std::vector<int32_t> cEnd(std::max<size_t>(rlen.size(), 1)), bEnd(std::max<size_t>(qs.size(), 1));
      int32_t nc = 0, nb = 0;
      check(bani_ctx_plan_run(ctx, 0, 0, rlen.data(), rcont.data(), (int32_t)rlen.size(), qlen.data(), nullptr, (int32_t)qs.size(),
                              cEnd.data(), &nc, bEnd.data(), &nb, &indexBudget), "bani_ctx_plan_run");
      if (nc > 0) { chunks.clear(); for (int32_t c = 0, a = 0; c < nc; a = cEnd[c], c++) chunks.push_back({a, cEnd[c]}); }
      if (nb > 0) { blocks.clear(); for (int32_t c = 0, a = 0; c < nb; a = bEnd[c], c++) blocks.push_back({a, bEnd[c]}); }
      {
        std::lock_guard<std::mutex> l(mu);
        std::cerr << "INFO [GPU " << g << "], skch::main, " << (loading ? "shard file " + std::to_string(s) + ", " : std::string())
                  << "reference chunks : " << chunks.size() << ", query blocks : " << blocks.size() << " (index budget " << indexBudget << " bytes)" << std::endl;
      }
      // member sketches of another block range than this shard's first block would only take device memory from its index
      if (memberCache[g].q0 != blocks[0].first || memberCache[g].q1 != blocks[0].second) memberCache[g].clear();
      if (chunks.size() > 1 || blocks.size() > 1) {
        if (parameters.visualize)
          throw std::runtime_error("--visualize needs the reference shard of a GPU in one index, this run needs " + std::to_string(chunks.size()) +
                                   " chunk(s) and " + std::to_string(blocks.size()) + " query block(s) on GPU " + std::to_string(g) + ": use more GPUs or fewer references");
        if (!parameters.saveIndex.empty())
          throw std::runtime_error("--saveIndex writes one index per GPU, this run needs " + std::to_string(chunks.size()) + " chunk(s) and " +
                                   std::to_string(blocks.size()) + " query block(s) on GPU " + std::to_string(g) + ": use more GPUs or fewer references");
        std::vector<cgi::CGI_Results> local;
        chunkedShard(ctx, g, s, shards[s], chunks, blocks, indexBudget, local);
        if (g == 0) std::cerr << "INFO [GPU 0], skch::main, Time spent " << (loading ? "loading" : "sketching") << " and mapping in chunks : "
                              << std::chrono::duration<double>(Clock::now() - t1).count() << " sec" << std::endl;
        cgi::correctRefGenomeIds(local, s, S, (int)parameters.refSequences.size(), parameters.blockPartition);
        std::lock_guard<std::mutex> l(mu);
        finalResults.insert(finalResults.end(), local.begin(), local.end());
        return;
      }
      // genomes this device needs: its reference shard (unless loaded) and every query that has to be read, each file once
      std::vector<int> need; std::unordered_map<int, int> slot;
      auto want = [&](const std::string &path) { const int id = pathId.at(path); if (!slot.count(id)) { slot[id] = (int)need.size(); need.push_back(id); } return slot[id]; };
      std::vector<int> refSlot, qrySlot;                              // qrySlot: -1 = derived from the index
      if (!loading) for (int j : shards[s]) refSlot.push_back(want(parameters.refSequences[j]));
      for (size_t q = 0; q < qs.size(); q++) qrySlot.push_back(derivable(q) ? -1 : want(qs[q]));
      std::vector<const bani_host::HostGenome *> hs; for (int id : need) hs.push_back(&genomes[id]);
      std::vector<std::unique_ptr<DeviceGenome>> dev;
      upload_genomes(ctx, hs, dev, (size_t)1 << 28, std::max(1, parameters.threads / G));
      std::vector<std::string> shardRefNames;
      for (int j : shards[s]) shardRefNames.push_back(parameters.refSequences[j]);

      std::unique_ptr<Sketch> referSketchP;                           // HP1, or the cache
      if (loading) referSketchP.reset(new Sketch(ctx, parameters, shardFile(parameters.loadIndex, s, S), meta.contigNames[s]));
      else {
        std::vector<const DeviceGenome *> refs;
        for (int sl : refSlot) refs.push_back(dev[sl].get());
        referSketchP.reset(new Sketch(ctx, parameters, refs));
      }
      Sketch &referSketch = *referSketchP;
      if (g == 0) std::cerr << "INFO [GPU 0], skch::main, Time spent " << (loading ? "loading" : "sketching") << " the reference : "
                            << std::chrono::duration<double>(Clock::now() - t1).count() << " sec" << std::endl;
      if (!parameters.saveIndex.empty()) {
        referSketch.save(shardFile(parameters.saveIndex, s, S));
        for (const auto &c : referSketch.metadata) savedContigNames[s].push_back(c.name);
      }
      std::vector<cgi::CGI_Results> local;
      sanity[s] = referSketch.sanityCheck(parameters.maxRatioDiff); ratioDiffs[s] = referSketch.getRatioDifference();
      if (sanity[s]) {
        t1 = Clock::now();
        if (hostCgi) {
          std::ostringstream vis;
          for (size_t q = 0; q < qrySlot.size(); q++) {
            MappingResultsVector_t mapResults; uint64_t totalQueryFragments = 0;
            Map mapper(ctx, parameters, referSketch, *dev[qrySlot[q]], totalQueryFragments,
                       std::bind(Map::insertL2ResultsToVec, std::ref(mapResults), std::placeholders::_1));     // HP2
            cgi::computeCGI(parameters, mapResults, mapper, referSketch, totalQueryFragments, q, parameters.querySequences[q],
                            shardRefNames, &vis, local);
          }
          visual[s] = vis.str();
        } else {
          // HP2 + reduction for all queries: one sketch object for the queries that were read, and those derived -- from
          // the loaded index itself when it is the only shard, else one per shard file that holds members (kept for the
          // GPU's next shard file)
          std::vector<bani_genome *> qh; std::vector<int32_t> qid, dord, did;
          for (size_t q = 0; q < qrySlot.size(); q++) {
            if (qrySlot[q] >= 0) { qh.push_back(dev[qrySlot[q]]->h); qid.push_back((int32_t)q); }
            else { dord.push_back(memberAt[q].second); did.push_back((int32_t)q); }
          }
          std::vector<bani_qsketch *> sk;
          if (!qh.empty()) { bani_qsketch *x = nullptr; check(bani_qsketch_create(ctx, qh.data(), (int32_t)qh.size(), qid.data(), referSketch.handle(), &x), "bani_qsketch_create"); sk.push_back(x); }
          if (!dord.empty() && S == 1) { bani_qsketch *x = nullptr; check(bani_qsketch_from_index(ctx, referSketch.handle(), dord.data(), (int32_t)dord.size(), did.data(), &x), "bani_qsketch_from_index"); sk.push_back(x); }
          const size_t owned = sk.size();
          if (!dord.empty() && S > 1) { const auto &m = memberSketches(ctx, g, 0, (int)qs.size()); sk.insert(sk.end(), m.begin(), m.end()); }
          bani_cgi_result *res = nullptr; uint64_t n = 0; bani_map_counters ctr;
          bani_frag_mapping *frags = nullptr; uint64_t nf = 0;
          const int rc = parameters.visualize                                                                  // HP2 + reduction
            ? bani_map_cgi_sketch_frags(ctx, referSketch.handle(), sk.data(), (int32_t)sk.size(), &res, &n, &frags, &nf, &ctr)
            : bani_map_cgi_sketch(ctx, referSketch.handle(), sk.data(), (int32_t)sk.size(), &res, &n, &ctr);
          for (size_t i = 0; i < owned; i++) bani_qsketch_destroy(sk[i]);
          check(rc, parameters.visualize ? "bani_map_cgi_sketch_frags" : "bani_map_cgi_sketch");
          for (uint64_t i = 0; i < n; i++)
            local.push_back(cgi::CGI_Results{res[i].refGenomeId, res[i].qryGenomeId, res[i].countSeq, res[i].totalQueryFragments, res[i].identity});
          bani_free(res);
          if (parameters.visualize) {
            // frags come per sketch (queries read, then queries derived): .visual lines go in query-list order.  The
            // frags of one query are contiguous and in bin order, so a stable sort by query keeps that order.
            std::stable_sort(frags, frags + nf, [](const bani_frag_mapping &a, const bani_frag_mapping &b) { return a.qryGenomeId < b.qryGenomeId; });
            std::vector<skch::offset_t> refLens;
            for (const auto &c : referSketch.metadata) refLens.push_back(c.len);
            const std::vector<int64_t> refOff = cgi::offsetAdder(refLens);
            std::ostringstream vis;
            for (uint64_t i = 0; i < nf;) {
              const int32_t q = frags[i].qryGenomeId;
              uint64_t j = i;
              while (j < nf && frags[j].qryGenomeId == q) j++;
              // Map::metadata of the query: from its file, or (derived query) from its contigs in the shard file that holds it
              std::vector<skch::offset_t> qLens;
              if (qrySlot[q] >= 0) {
                for (const auto &c : dev[qrySlot[q]]->host->contigs) appendFragmentLengths(parameters, (offset_t)c.len, qLens);
              } else {
                const IndexFileTables &t = fileTables[memberAt[q].first];
                const int o = memberAt[q].second, c0 = o ? t.seqsByFile[o - 1] : 0, c1 = t.seqsByFile[o];
                for (int c = c0; c < c1; c++) appendFragmentLengths(parameters, t.contigLen[c], qLens);
              }
              cgi::outputVisualizationFile(parameters, frags + i, j - i, cgi::offsetAdder(qLens), refOff, referSketch,
                                           parameters.querySequences[q], shardRefNames, vis);
              i = j;
            }
            visual[s] = vis.str();
          }
          bani_free(frags);
        }
        if (g == 0) std::cerr << "INFO [GPU 0], skch::main, Time spent mapping " << qrySlot.size() << " query genome(s) : "
                              << std::chrono::duration<double>(Clock::now() - t1).count() << " sec" << std::endl;
      }
      cgi::correctRefGenomeIds(local, s, S, (int)parameters.refSequences.size(), parameters.blockPartition);
      std::lock_guard<std::mutex> l(mu);
      finalResults.insert(finalResults.end(), local.begin(), local.end());
    };

    auto gpuWork = [&](int g) {
      try {
        for (int s = g; s < S; s += G) shardRun(ctxs[g], g, s);
        memberCache[g].clear();
        if (getenv("BANI_CLI_FULL_TEARDOWN")) bani_ctx_destroy(ctxs[g]);      // otherwise the process exit returns the device memory (faster)
      } catch (const std::exception &e) { memberCache[g].clear(); std::lock_guard<std::mutex> l(mu); err = e.what(); }
    };
    {
      std::vector<std::thread> th;
      for (int g = 0; g < G; g++) th.emplace_back(gpuWork, g);
      for (auto &t : th) t.join();
    }
    if (!err.empty()) throw std::runtime_error(err);
    if (!parameters.saveIndex.empty()) writeMeta(parameters.saveIndex, parameters, S, savedContigNames);
    for (int s = 0; s < S; s++) {
      if (!sanity[s]) std::cerr << "ERROR :: SPLIT " << s << "'s ratio difference " << ratioDiffs[s] << " exceeds maximum thresholds." << std::endl;
      for (const auto &m : chunkSanity[s]) std::cerr << m << std::endl;
    }
    // a query derived from the index has the length its reference twin has
    for (const auto &q : parameters.querySequences) if (!genomeLengths.count(q)) throw std::runtime_error("no length known for " + q);

    cgi::outputCGI(parameters, genomeLengths, finalResults, fileName);
    if (parameters.matrixOutput) cgi::outputPhylip(parameters, genomeLengths, finalResults, fileName);
    if (parameters.visualize) { std::ofstream o(fileName + ".visual"); for (int s = 0; s < S; s++) o << visual[s]; }
    std::cerr << "INFO, skch::main, Total time : " << std::chrono::duration<double>(Clock::now() - tStart).count() << " sec" << std::endl;
  } catch (const std::exception &e) {
    std::cerr << "ERROR, " << e.what() << std::endl;
    return 1;
  }
  std::cout.flush(); std::cerr.flush();
  if (!getenv("BANI_CLI_FULL_TEARDOWN")) _exit(0);      // outputs are written and closed: skip the destructors of multi-GB host tables and the CUDA teardown
  return 0;
}
