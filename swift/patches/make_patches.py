#!/usr/bin/env python
"""Generates swift/patches/*.patch: the call-site re-point of SURVEY.md section 8(f1) as unified diffs against the
reference tree (a checkout of christopherkarani/Wax at the surveyed revision).

    python swift/patches/make_patches.py <path to the Wax checkout>

What the patches do (nothing else of Wax is touched):
  * every closed enum that selects a vector engine gains `case cuda(CUDAVectorEngine)` under
    `#if canImport(WaxVectorSearchCUDAC)`, and the Metal case moves under `#if canImport(Metal)` so the same sources
    build on Linux (where Metal does not exist and the CUDA C module does);
  * engine selection tries CUDA first (`CUDAVectorEngine.isAvailable`), then Metal, then USearch, with the
    reference's own "log and fall back" behaviour (WaxSession.swift:484-497);
  * WaxSession.search hands its resident engine to the unified search instead of `nil`, so a store is not held twice
    (15 GB at 10 M rows) -- SURVEY.md section 3.1;
  * Package.swift gains the C module target `WaxVectorSearchCUDAC` (header + modulemap + `-lwaxvs_cuda`), Linux only,
    following the WaxCoreCompressionC precedent (Package.swift:54-73).

The patches are mechanical rewrites of short, regular code (one-line switch arms); they are NOT compiled (the project is built
without a Swift toolchain); `git apply --check` against a Wax checkout shows that each applies cleanly."""
from __future__ import annotations

import difflib
import re
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
if len(sys.argv) != 2:
    sys.exit("usage: python swift/patches/make_patches.py <path to a Wax checkout>")
REF = Path(sys.argv[1])
CUDA_IF, METAL_IF, ENDIF = "#if canImport(WaxVectorSearchCUDAC)", "#if canImport(Metal)", "#endif"


def guard_switch_arms(src: str) -> str:
    """`case .metal(let engine): <one line>` -> the same arm under canImport(Metal) + a `.cuda` twin."""
    pat = re.compile(r"^(?P<i>[ \t]*)case \.metal\(let engine\):\n(?P<body>[ \t]*[^\n]*\n)", re.M)

    def sub(m):
        i, body = m.group("i"), m.group("body")
        return (f"{i}{METAL_IF}\n{i}case .metal(let engine):\n{body}{i}{ENDIF}\n"
                f"{i}{CUDA_IF}\n{i}case .cuda(let engine):\n{body}{i}{ENDIF}\n")
    return pat.sub(sub, src)


def guard_enum_case(src: str) -> str:
    pat = re.compile(r"^(?P<i>[ \t]*)case metal\(MetalVectorEngine\)\n", re.M)
    return pat.sub(lambda m: (f"{m.group('i')}{METAL_IF}\n{m.group('i')}case metal(MetalVectorEngine)\n{m.group('i')}{ENDIF}\n"
                              f"{m.group('i')}{CUDA_IF}\n{m.group('i')}case cuda(CUDAVectorEngine)\n{m.group('i')}{ENDIF}\n"), src)


def must_replace(src: str, old: str, new: str) -> str:
    assert src.count(old) == 1, f"expected exactly one occurrence of:\n{old}"
    return src.replace(old, new)


def patch_wax_session(src: str) -> str:
    src = guard_switch_arms(guard_enum_case(src))
    src = must_replace(src, """            textEngine: textEngine,
            vectorEngine: nil,
""", """            textEngine: textEngine,
            vectorEngine: vectorEngine,
""")
    return must_replace(src, """        if preference != .cpuOnly, MetalVectorEngine.isAvailable {
            do {
                let metal = try await MetalVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
                return .metal(metal)
            } catch {
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "metal vector engine load",
                    fallback: "use CPU vector engine"
                )
            }
        }
""", f"""        {CUDA_IF}
        if preference != .cpuOnly, CUDAVectorEngine.isAvailable {{
            do {{
                let cuda = try await CUDAVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
                return .cuda(cuda)
            }} catch {{
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "cuda vector engine load",
                    fallback: "use the next vector engine"
                )
            }}
        }}
        {ENDIF}
        {METAL_IF}
        if preference != .cpuOnly, MetalVectorEngine.isAvailable {{
            do {{
                let metal = try await MetalVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
                return .metal(metal)
            }} catch {{
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "metal vector engine load",
                    fallback: "use CPU vector engine"
                )
            }}
        }}
        {ENDIF}
""")


def patch_vector_search_session(src: str) -> str:
    src = guard_switch_arms(guard_enum_case(src))
    return must_replace(src, """        let loadedEngine: ConcreteVectorEngine
        if preference != .cpuOnly, MetalVectorEngine.isAvailable {
            // Try Metal first; if load fails, fall back to CPU without aborting the session.
            do {
                let metal = try await MetalVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
                loadedEngine = .metal(metal)
            } catch {
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "metal vector engine load",
                    fallback: "use CPU vector engine"
                )
                let usearch = try await USearchVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
                loadedEngine = .usearch(usearch)
            }
        } else {
            let usearch = try await USearchVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
            loadedEngine = .usearch(usearch)
        }
""", f"""        // GPU engines first (CUDA, then Metal); a failed load falls back to the CPU engine without aborting the session.
        var gpuEngine: ConcreteVectorEngine?
        {CUDA_IF}
        if gpuEngine == nil, preference != .cpuOnly, CUDAVectorEngine.isAvailable {{
            do {{
                gpuEngine = .cuda(try await CUDAVectorEngine.load(from: wax, metric: metric, dimensions: dimensions))
            }} catch {{
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "cuda vector engine load",
                    fallback: "use the next vector engine"
                )
            }}
        }}
        {ENDIF}
        {METAL_IF}
        if gpuEngine == nil, preference != .cpuOnly, MetalVectorEngine.isAvailable {{
            do {{
                gpuEngine = .metal(try await MetalVectorEngine.load(from: wax, metric: metric, dimensions: dimensions))
            }} catch {{
                WaxDiagnostics.logSwallowed(
                    error,
                    context: "metal vector engine load",
                    fallback: "use CPU vector engine"
                )
            }}
        }}
        {ENDIF}
        let loadedEngine: ConcreteVectorEngine
        if let gpuEngine {{
            loadedEngine = gpuEngine
        }} else {{
            let usearch = try await USearchVectorEngine.load(from: wax, metric: metric, dimensions: dimensions)
            loadedEngine = .usearch(usearch)
        }}
""")


def patch_engine_cache(src: str) -> str:
    src = must_replace(src, """        case usearch
        case metal
    }
""", f"""        case usearch
        case metal
        case cuda
    }}
""")
    src = must_replace(src, """        let allowMetal = preference != .cpuOnly && MetalVectorEngine.isAvailable

        if allowMetal {
""", f"""        {CUDA_IF}
        if preference != .cpuOnly && CUDAVectorEngine.isAvailable {{
            if let cudaEngine = try await vectorEngine(
                for: wax,
                waxId: waxId,
                queryEmbeddingDimensions: queryEmbeddingDimensions,
                engineKind: .cuda
            ) {{
                return cudaEngine
            }}
        }}
        {ENDIF}
        {METAL_IF}
        let allowMetal = preference != .cpuOnly && MetalVectorEngine.isAvailable
        #else
        let allowMetal = false
        {ENDIF}

        if allowMetal {{
""")
    src = must_replace(src, """        let preferMetal = engineKind == .metal

        let makeEngine: (VectorMetric, Int) throws -> any VectorSearchEngine = { metric, dimensions in
            if preferMetal {
                return try MetalVectorEngine(metric: metric, dimensions: dimensions)
            }
            return try USearchVectorEngine(metric: metric, dimensions: dimensions)
        }
""", f"""        let makeEngine: (VectorMetric, Int) throws -> any VectorSearchEngine = {{ metric, dimensions in
            switch engineKindTag {{
            case .metal:
                {METAL_IF}
                return try MetalVectorEngine(metric: metric, dimensions: dimensions)
                #else
                throw WaxError.invalidToc(reason: "metal engine not available on this platform")
                {ENDIF}
            case .cuda:
                {CUDA_IF}
                return try CUDAVectorEngine(metric: metric, dimensions: dimensions)
                #else
                throw WaxError.invalidToc(reason: "cuda engine not available on this platform")
                {ENDIF}
            case .usearch:
                return try USearchVectorEngine(metric: metric, dimensions: dimensions)
            }}
        }}
""")
    return must_replace(src, """            case .metal:
                guard let metal = engine as? MetalVectorEngine else {
                    throw WaxError.invalidToc(reason: "metal engine type mismatch")
                }
                try await metal.deserialize(bytes)
""", f"""            case .metal:
                {METAL_IF}
                guard let metal = engine as? MetalVectorEngine else {{
                    throw WaxError.invalidToc(reason: "metal engine type mismatch")
                }}
                try await metal.deserialize(bytes)
                #else
                throw WaxError.invalidToc(reason: "metal engine not available on this platform")
                {ENDIF}
            case .cuda:
                {CUDA_IF}
                guard let cuda = engine as? CUDAVectorEngine else {{
                    throw WaxError.invalidToc(reason: "cuda engine type mismatch")
                }}
                try await cuda.deserialize(bytes)
                #else
                throw WaxError.invalidToc(reason: "cuda engine not available on this platform")
                {ENDIF}
""")


def patch_unified_search(src: str) -> str:
    # The Metal kernel assumes a unit query (VectorMath.isNormalizedL2 tolerance 1e-3); the CUDA kernel always divides by
    # the real |q|, so it needs no host-side normalisation: only the platform guard changes here.
    return must_replace(src, """            if vectorEngine is MetalVectorEngine, !VectorMath.isNormalizedL2(queryEmbedding) {
                queryEmbedding = VectorMath.normalizeL2(queryEmbedding)
            }
""", f"""            {METAL_IF}
            if vectorEngine is MetalVectorEngine, !VectorMath.isNormalizedL2(queryEmbedding) {{
                queryEmbedding = VectorMath.normalizeL2(queryEmbedding)
            }}
            {ENDIF}
""")


def patch_package(src: str) -> str:
    src = must_replace(src, """        .target(
            name: "WaxVectorSearch",
            dependencies: [
                "WaxCore",
                .product(name: "USearch", package: "USearch"),
            ],
""", """        .target(
            name: "WaxVectorSearchCUDAC",
            dependencies: [],
            path: "Sources/WaxVectorSearchCUDAC",
            publicHeadersPath: "include",
            linkerSettings: [
                .linkedLibrary("waxvs_cuda", .when(platforms: [.linux])),
            ]
        ),
        .target(
            name: "WaxVectorSearch",
            dependencies: [
                "WaxCore",
                .product(name: "USearch", package: "USearch"),
                .target(
                    name: "WaxVectorSearchCUDAC",
                    condition: .when(platforms: [.linux])
                ),
            ],
""")
    return src


TARGETS = {
    "Sources/Wax/WaxSession.swift": patch_wax_session,
    "Sources/Wax/VectorSearchSession.swift": patch_vector_search_session,
    "Sources/Wax/UnifiedSearch/UnifiedSearchEngineCache.swift": patch_engine_cache,
    "Sources/Wax/UnifiedSearch/UnifiedSearch.swift": patch_unified_search,
    "Package.swift": patch_package,
}


def main() -> None:
    for rel, fn in TARGETS.items():
        old = (REF / rel).read_text()
        new = fn(old)
        assert new != old, rel
        diff = "".join(difflib.unified_diff(old.splitlines(True), new.splitlines(True), f"a/{rel}", f"b/{rel}", n=2))
        out = HERE / (rel.replace("/", "__") + ".patch")
        out.write_text(diff)
        print(f"{out.name}: +{sum(1 for l in diff.splitlines() if l.startswith('+') and not l.startswith('+++'))} "
              f"-{sum(1 for l in diff.splitlines() if l.startswith('-') and not l.startswith('---'))}")


if __name__ == "__main__":
    main()
